"""GPU: triangle-mesh bodies (DESIGN.md §8, "Mesh bodies").  Box and sphere bodies set through blub_fluid_set_bodies_meshes equal the same
set through blub_fluid_set_bodies; cleared mesh bodies leave no trace; the composite volume, marker, load sums and integration of an
icosphere, a torus and an L-block agree bit for bit with tests/mesh_body_ref.py; a 12-triangle box mesh is the box body; every recorded pose
is the restated integration of the previous one; an L-block rests on its lowest corner; an icosphere and a hollow hull denser than the fluid
float at the predicted draft; runs are reproducible; refusals change nothing."""
import numpy as np
import pytest
from scipy.optimize import brentq

import blub_b200
from blub_b200 import fluid as F
from tests import body_ref, mesh_body_ref as M, util
from tests.test_gpu_bodies import DOUBLE_DAM_BODIES, INV_DT, SCENE_G, S30, pose, record, surface
from tests.test_gpu_loads import BOX, Solid, seed_around
from tests.test_gpu_state import snapshot
from tests.test_gpu_tags import assert_same_physics, bits
from tests.util import DT

pytestmark = pytest.mark.gpu

TILT = (float(np.float32(np.cos(0.3))), float(np.float32(np.sin(0.3) * 0.6)), 0.0, float(np.float32(np.sin(0.3) * 0.8)))
ICO, TORUS, LBLOCK = M.icosphere(2, 1.0), M.torus(2.0, 0.8, 24, 12), M.l_block()
# (mesh, scale, placement) on double_dam, clear of the moving box and the walls
MESH_BODIES = [(ICO, 5.0, body_ref.body("box", 1, 0.6, (110, 22, 20), TILT, (0, 0, 0), (0, 0.4, 0))),
               (TORUS, 3.0, body_ref.body("box", 1, 0.8, (22, 30, 50), S30, (1, 0, 0))),
               (LBLOCK, 3.0, body_ref.body("box", 1, 0.7, (104, 26, 46), TILT, (0, 0, 0), (0.2, 0, 0)))]


def mesh_dicts(spec):
    return [dict(b, shape="mesh", mesh=mesh, scale=s) for mesh, s, b in spec]


def restated(f, spec):
    """(per-body (mid, body-frame vertices, triangles) or None, per-body (mass, moments, mid) or None, the set's cube side)."""
    meshes, masses, mids = [], [], []
    for i, item in enumerate(spec):
        if item is None:
            meshes.append(None), masses.append(None), mids.append(None)
            continue
        (pos, tri), scale = item[0], item[1]
        p = f.body_mass_properties(i)
        mid, _ = M.mid_and_half(p)
        meshes.append((mid, F.mesh_body_vertices(pos, tri, scale), tri))
        masses.append((p["mass"], p["moments"], mid))
        mids.append(mid)
    return meshes, masses, M.cube_side(f.bodies(), mids)


def set_raw(f, bodies, meshes):
    """blub_fluid_set_bodies_meshes through ctypes: meshes[i] = (F.Mesh, scale) or None."""
    n = len(bodies)
    arr = (F.Body * max(n, 1))()
    shapes = (F.MeshBodyShape * max(n, 1))()
    for k, b in enumerate(bodies):
        arr[k] = F.Body.from_dict(b)
        if meshes[k] is not None:
            shapes[k].mesh, shapes[k].scale = meshes[k][0].h, meshes[k][1]
    return f.L.blub_fluid_set_bodies_meshes(f.h, arr, shapes, n)


# ---- 1. nothing changes without mesh bodies ------------------------------------------------------------------------------------
def test_null_meshes_equal_set_bodies():
    runs = []
    for raw in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
        if raw:
            assert set_raw(f, DOUBLE_DAM_BODIES, [None, None]) == F.BLUB_OK
        else:
            f.set_bodies(DOUBLE_DAM_BODIES)
        for _ in range(30):
            f.step(DT)
        runs.append((snapshot(f), [f.body_history(i) for i in range(2)]))
    assert_same_physics(runs[0][0], runs[1][0], stats=False)
    for ha, hb in zip(runs[0][1], runs[1][1]):
        for name in ha:
            assert np.array_equal(ha[name], hb[name]), name


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_cleared_mesh_bodies_change_nothing(tmp_path, path, graph):
    runs = []
    for had in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        if had:
            f.set_bodies(mesh_dicts([(ICO, 4.0, body_ref.body("box", 1, 0.5, (16, 20, 16)))]) + [body_ref.body("sphere", 3, 2.0, (8, 8, 8))])
            f.set_bodies([])
        for _ in range(70):
            f.step(DT)
            f.synchronize()
        save = str(tmp_path / f"{int(had)}.blub")
        f.save_state(save)
        runs.append((snapshot(f), open(save, "rb").read()))
    assert_same_physics(runs[0][0], runs[1][0])
    assert np.array_equal(bits(runs[0][0]["particles_position"]), bits(runs[1][0]["particles_position"]))
    assert runs[0][1] == runs[1][1]


# ---- 2. composite volume, marker, loads and integration bit for bit ---------------------------------------------------------------
def test_composite_marker_loads_and_integration_match_the_restatement(tmp_path):
    import torch
    f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    solid = Solid(f, BOX)
    f.set_bodies(mesh_dicts(MESH_BODIES))
    dims = f.grid_dimension()
    meshes, masses, cube = restated(f, MESH_BODIES)
    for _ in range(12):
        solid.step()
    before = f.bodies()
    assert [b["shape"] for b in before] == ["mesh"] * 3
    solid.voxelize()
    f.step_stages(DT, 0, 1)
    borrowed = solid.vol.cpu().numpy()
    want = M.composite(dims, borrowed, before, meshes, cube)
    got = f.download_solid_voxels()
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    for i, b in enumerate(before):  # every body covers cells, and no cell centre inside its mesh is missed
        mask, _ = M.covered(dims, b, meshes[i], cube)
        assert mask.sum() > 50, i
    # the marker: a twin with the restated composite volume as its borrowed one and no bodies
    twin = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    tsolid = Solid(twin, BOX)
    for _ in range(12):
        tsolid.step()
    # the twin's particles differ (its solids differed): compare the marker's SOLID cells, which depend on the volume alone
    vol = torch.from_numpy(want).cuda()
    torch.cuda.synchronize()
    twin.set_solid_voxels(vol.data_ptr())
    twin.step_stages(DT, 0, 1)
    solid_f, solid_t = f.download_grid(F.TAP_MARKER) == body_ref.SOLID, twin.download_grid(F.TAP_MARKER) == body_ref.SOLID
    assert np.array_equal(solid_f, solid_t)
    twin.step_stages(DT, 1, 14)
    f.step_stages(DT, 1, 3)
    marker, p_vel = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_P_VEL)
    for i, b in enumerate(before):
        h = f.body_history(i, 1)
        assert h["step"].tolist() == [12]
        assert record(h) == M.loads(marker, p_vel, INV_DT, b, meshes[i], cube), i
        assert record(h)["wetted_faces"] > 0
        want_pose = M.integrate(b, h["force_fx"][-1], h["torque_fx"][-1], DT, SCENE_G, dims, *masses[i])
        for name, v in pose(h).items():
            assert np.array_equal(np.float32(v), np.float32(want_pose[name])), (i, name)
    f.step_stages(DT, 3, 14)


def test_a_box_mesh_is_the_box_body():
    """The 12-triangle box mesh of half extents (4, 3, 5) at a pose with no cell centre within 1e-3 of a face writes the box body's
    composite volume and first-step sums bit for bit."""
    h = (4.0, 3.0, 5.0)
    mesh = M.box_mesh([-v for v in h], h)
    q = TILT
    c = (100.3, 21.37, 30.21)
    runs = []
    for as_mesh in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
        b = body_ref.body("box", h, 0.6, c, q)
        f.set_bodies(mesh_dicts([(mesh, 1.0, b)]) if as_mesh else [b])
        if as_mesh:
            p = f.body_mass_properties(0)
            assert p["principal_rotation"] == (1.0, 0.0, 0.0, 0.0) and p["centroid"] == (0.0, 0.0, 0.0)
            assert f.bodies()[0]["centre"] == body_ref.body("box", h, 0.6, c, q)["centre"]
        f.step_stages(DT, 0, 1)
        vol = f.download_solid_voxels()
        f.step_stages(DT, 1, 14)
        runs.append((vol, record(f.body_history(0, 1))))
    # the restated box body: no cell centre within 1e-3 of a face
    b = body_ref.body("box", h, 0.6, c, q)
    dims = (128, 64, 64)
    _, d = body_ref.covered(dims, b)
    R = body_ref.rotation(b["rotation"])
    u = [body_ref.dot3(R[0][j], R[1][j], R[2][j], d[0], d[1], d[2]) for j in range(3)]
    for j in range(3):  # the cells next to face j: within the face's extent in the other two body coordinates
        near = np.ones(u[0].shape, dtype=bool)
        for k in range(3):
            if k != j:
                near &= np.abs(u[k]) <= h[k] + 0.01
        assert np.abs(np.abs(u[j][near]) - np.float32(h[j])).min() > 1e-3
    assert np.array_equal(runs[0][0].view(np.uint16), runs[1][0].view(np.uint16))
    assert runs[0][1] == runs[1][1] and runs[0][1]["wetted_faces"] > 0


# ---- 3. the integrator over a run ------------------------------------------------------------------------------------------------
def test_every_recorded_pose_is_the_restated_integration_of_the_previous_one():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    f.set_bodies(mesh_dicts(MESH_BODIES))
    dims = f.grid_dimension()
    _, masses, _ = restated(f, MESH_BODIES)
    prev = f.bodies()
    for step in range(200):
        f.step(DT)
        for i in range(len(prev)):
            h = f.body_history(i, 1)
            assert h["step"].tolist() == [step]
            want = M.integrate(prev[i], h["force_fx"][-1], h["torque_fx"][-1], DT, SCENE_G, dims, *masses[i])
            for name, v in pose(h).items():
                assert np.array_equal(np.float32(v), np.float32(want[name])), (step, i, name)
        prev = f.bodies()
    assert max(abs(b["velocity"][1]) for b in prev) > 0.0


def test_an_l_block_falls_to_rest_on_its_lowest_corner():
    f = blub_b200.HybridFluid(64, 64, 64, 1000)
    g = (0.0, -981.0, 0.0)
    f.set_gravity_grid(g)
    f.set_bodies(mesh_dicts([(LBLOCK, 4.0, body_ref.body("box", 1, 0.7, (30, 40, 30), TILT))]))
    p = f.body_mass_properties(0)
    mid, half = M.mid_and_half(p)
    for _ in range(80):
        f.step(DT)
    b = f.bodies()[0]
    R = body_ref.rotation(b["rotation"])
    e = body_ref.bounding_extents(dict(b, shape="box"), R)
    off = M.box_offset(R, mid)
    lowest = (np.float32(b["centre"][1]) + off[1]) - e[1]
    assert abs(float(lowest) - 1.0) < 1e-5 and b["velocity"][1] == 0.0
    assert b["centre"][1] != float(np.float32(1) + e[1])  # not the symmetric bound a box body would rest on
    # no vertex below the floor
    vg = M.grid_vertices(b, F.mesh_body_vertices(*LBLOCK, 4.0))
    assert float(vg[:, 1].min()) >= 1.0 - 1e-5


# ---- 4. Archimedes, and a hollow hull -------------------------------------------------------------------------------------------
def test_a_floating_icosphere_finds_the_discrete_hydrostatic_draft():
    """rho_r 0.5, radius 5 cells: it floats with the displaced volume half its own.  The prediction counts the cells whose centre lies
    inside the sphere below the discrete surface (the cells the body covers at its pose)."""
    r, rho = 5.0, 0.5
    f = blub_b200.HybridFluid(64, 64, 64, 8 * 64 * 64 * 32)
    f.set_gravity_grid((0.0, -981.0, 0.0))
    seed_around(f, 33, (26, 27, 26), (38, 33, 38))  # no particle starts inside the sphere
    for which in (0, 1):
        f.set_solver_config(which, 1e-5, 4000, 4)
    f.set_bodies(mesh_dicts([(M.icosphere(3, 1.0), r, body_ref.body("box", 1, rho, (32, 33, 32)))]))
    meshes = M.icosphere(3, 1.0)
    vb = F.mesh_body_vertices(*meshes, r)
    drafts = []
    for step in range(400):
        f.step(DT)
        if step >= 300:
            b = f.bodies()[0]
            s = surface(f.download_grid(F.TAP_MARKER), b["centre"][0], b["centre"][2])
            drafts.append(s - (b["centre"][1] + float(vb[:, 1].min())))
    # the prediction: the spherical cap holding rho V below the surface (depth r for rho 0.5), less one cell as for the box, whose discrete
    # draft is 8 rho - 1
    V = f.body_mass_properties(0)["volume"]
    depth = brentq(lambda h: np.pi * h * h * (3 * r - h) / 3 - rho * V, 0.0, 2 * r) - 1.0
    assert abs(np.mean(drafts) - depth) < 1.5, (np.mean(drafts), depth, drafts[::10])


def test_a_hollow_hull_denser_than_the_fluid_floats():
    """A 20-cell box with a cavity open at the top, walls and floor 2 cells thick, rho_r 1.5: mass / outer volume = 1.5 * 3392 / 8000 = 0.64,
    so it floats, with the cavity dry, although its material is denser than the fluid."""
    outer, wall, rho = 20, 2, 1.5
    pos, tri = M.hollow_box(outer, wall)
    f = blub_b200.HybridFluid(64, 64, 64, 8 * 64 * 64 * 32)
    f.set_gravity_grid((0.0, -981.0, 0.0))
    lo, hi = (22, 20, 22), (42, 40, 42)
    seed_around(f, 33, lo, (hi[0], 33, hi[2]))  # no particle starts inside the hull or its cavity
    for which in (0, 1):
        f.set_solver_config(which, 1e-5, 4000, 4)
    f.set_bodies(mesh_dicts([((pos, tri), 1.0, body_ref.body("box", 1, rho, lo))]))
    p = f.body_mass_properties(0)
    assert abs(p["volume"] - (outer ** 3 - (outer - 2 * wall) ** 2 * (outer - wall))) < 1e-6
    vb = F.mesh_body_vertices(pos, tri, 1.0)
    drafts, wet = [], []
    for step in range(400):
        f.step(DT)
        if step >= 300:
            b = f.bodies()[0]
            marker = f.download_grid(F.TAP_MARKER)
            s = surface(marker, b["centre"][0], b["centre"][2])
            bottom = b["centre"][1] + float(vb[:, 1].min())
            drafts.append(s - bottom)
            cx, cz = int(b["centre"][0]), int(b["centre"][2])
            cav = marker[cz - 2:cz + 2, int(bottom) + wall + 1:int(bottom) + outer, cx - 2:cx + 2]
            wet.append(float((cav == 1).mean()))
    # the hull displaces its outer volume below the surface: draft = rho V / outer^2, less one cell as for the box
    want = rho * p["volume"] / outer ** 2 - 1.0
    assert abs(np.mean(drafts) - want) < 1.5, (np.mean(drafts), want, drafts[::10])
    assert np.mean(wet) < 0.2, wet[::10]


# ---- 5. reproducibility, refusals --------------------------------------------------------------------------------------------
def test_two_runs_and_graph_against_eager_are_bit_identical():
    runs = []
    for graph in (True, True, False):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
        f.set_graph_replay(graph)
        f.set_bodies(mesh_dicts(MESH_BODIES) + [DOUBLE_DAM_BODIES[1]])
        for _ in range(100):
            f.step(DT)
        runs.append((snapshot(f), [f.body_history(i) for i in range(4)]))
    for other in runs[1:]:
        assert_same_physics(runs[0][0], other[0], stats=False)
        for ha, hb in zip(runs[0][1], other[1]):
            for name in ha:
                assert np.array_equal(ha[name], hb[name]), name


def test_refusals_change_nothing(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    good = mesh_dicts([(ICO, 4.0, body_ref.body("box", 1, 0.5, (16, 20, 16)))])
    f.set_bodies(good)
    f.step(DT)
    before, hist = f.bodies(), f.body_history(0)
    pos, tri = ICO
    open_mesh = (pos, tri[1:])
    flipped = (pos, np.concatenate([tri[:1, ::-1], tri[1:]]))
    bad = [dict(good[0], mesh=open_mesh), dict(good[0], mesh=flipped), dict(good[0], scale=0.0), dict(good[0], scale=float("inf")),
           dict(good[0], scale=0.4), dict(good[0], centre=(3, 20, 16)), dict(good[0], relative_density=0.0)]
    for b in bad:
        with pytest.raises(F.BlubError):
            f.set_bodies([b])
    with pytest.raises(F.BlubError):  # over the total vertex limit: 16 copies of a 2^15-vertex sphere would be 2^19 vertices
        big = M.icosphere(6, 1.0)
        f.set_bodies([dict(good[0], mesh=big, centre=(16, 20, 16))] * 9)
    with pytest.raises(F.BlubError):
        f.body_mass_properties(1)
    assert f.bodies() == before and len(f.body_history(0)["step"]) == len(hist["step"])
    f.step(DT)
    assert len(f.body_history(0)["step"]) == 2


# ---- 6. checkpoint and the runner ----------------------------------------------------------------------------------------------
def test_a_saved_fluid_with_mesh_bodies_flow_and_tags_resumes_bit_for_bit(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    f.set_bodies(mesh_dicts([(LBLOCK, 2.0, body_ref.body("box", 1, 0.5, (18, 16, 14), S30))]) + [body_ref.body("sphere", 3, 1.5, (10, 24, 20))])
    f.paint_tags((1, 1, 1), (16, 31, 31), 7)
    for _ in range(20):
        f.step(DT)
    state = str(tmp_path / "s.blub")
    f.save_state(state)
    assert F.state_info(state).format_version == 16
    g = blub_b200.HybridFluid.from_state(state)
    pf, pg = f.body_mass_properties(0), g.body_mass_properties(0)
    for k in pf:
        assert np.array_equal(np.asarray(pf[k]), np.asarray(pg[k])), k
    assert g.bodies() == f.bodies()
    for _ in range(20):  # past the re-sorts of steps 24 and 32
        f.step(DT)
        g.step(DT)
    a, b = snapshot(f), snapshot(g)
    assert_same_physics(a, b, stats=False)
    assert np.array_equal(bits(a["particles_position"]), bits(b["particles_position"]))
    assert g.bodies() == f.bodies()
    for i in range(2):
        hf, hg = f.body_history(i, 20), g.body_history(i)
        for name in hf:
            assert np.array_equal(hf[name], hg[name]), name


def test_runner_mesh_bodies_equal_a_ctypes_run(tmp_path):
    import json
    import subprocess
    from tests.test_gpu_loads import RUNNER
    from tests.test_mesh_bodies_kat import write_obj
    sc = json.load(open(util.scene_path("dam_small")))
    v3 = lambda x, y, z: {"x": x, "y": y, "z": z}  # noqa: E731
    (tmp_path / "models").mkdir()
    write_obj(str(tmp_path / "models" / "l.obj"), *LBLOCK)
    sc["fluid"]["bodies"] = [{"shape": "mesh", "model": "models/l.obj", "scale": 0.02, "position": v3(0.1, 0.12, 0.16), "relative_density": 0.6,
                              "rotation_angles_deg": v3(0.0, 20.0, 0.0)},
                             {"shape": "sphere", "position": v3(0.24, 0.2, 0.16), "half_extent": 0.03, "relative_density": 1.5}]
    scene = str(tmp_path / "bodies.json")
    json.dump(sc, open(scene, "w"))
    steps = 1100
    out, out2, state = str(tmp_path / "o1.json"), str(tmp_path / "o2.json"), str(tmp_path / "s.blub")
    r = subprocess.run([RUNNER, scene, "--steps", str(steps), "--bodies", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([RUNNER, scene, "--steps", "600", "--save-state", state], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([RUNNER, scene, "--steps", str(steps - 600), "--load-state", state, "--bodies", out2], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    assert f.bodies()[0]["shape"] == "mesh"
    got = [[], []]
    for k in range(steps):
        f.step(DT)
        if (k + 1) % 500 == 0 or k + 1 == steps:
            for i in range(2):
                h = f.body_history(i)
                for j in range(len(h["step"])):
                    if not got[i] or h["step"][j] > got[i][-1]["step"]:
                        got[i].append({"step": int(h["step"][j]), "centre": [float(v) for v in h["centre"][j]],
                                       "rotation": [float(v) for v in h["rotation"][j]], "force": h["force"][j].tolist()})
    for run, first in ((json.load(open(out)), 0), (json.load(open(out2)), 600)):
        assert len(run["bodies"]) == 2
        for body, want in zip(run["bodies"], got):
            recs = body["records"]
            assert [r_["step"] for r_ in recs] == list(range(first, steps))
            for r_, w in zip(recs, want[first:]):
                assert np.array_equal(np.float32(r_["centre"]), np.float32(w["centre"])) and np.array_equal(np.float32(r_["rotation"]), np.float32(w["rotation"]))
                assert r_["force"] == w["force"]
