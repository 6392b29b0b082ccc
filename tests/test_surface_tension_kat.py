"""CPU: known answers of the surface tension rule (DESIGN.md §8 "Surface tension") through its NumPy restatement
tests/surface_tension_ref.py, the capillary step limit, the scene key and the version-64 state file as the host-only reader sees it.  No GPU
needed."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import cfl_ref, pcg_ref, surface_tension_ref as S, util
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_mesh_bodies_kat import v16_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes, write
from tests.test_viscosity_kat import viscosity_payload

BLUB_ERR_PARSE = 5
ONE = 1 << 40  # one particle weight in the splat's fixed point


def tank(shape):
    m = np.full(shape, S.AIR, dtype=np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def radial_splat(shape, centre, radius, kind="sphere", inside=True, width=8.0):
    """A sphere (or a cylinder along z) in the splat's fixed point: 8 particle weights deep inside, 0 far outside and a linear ramp in r of
    `width` cells across the surface (wide enough for every cell the band's curvature reads), and its marker."""
    z, y, x = np.indices(shape, dtype=np.float64) + 0.5
    d2 = (x - centre[2]) ** 2 + (y - centre[1]) ** 2 + (0.0 if kind == "cylinder" else (z - centre[0]) ** 2)
    r = np.sqrt(d2)
    level = np.clip(0.5 - (r - radius) / width, 0.0, 1.0)
    if not inside:
        level = 1.0 - level
    m = tank(shape)
    m[1:-1, 1:-1, 1:-1] = np.where(level[1:-1, 1:-1, 1:-1] > 0.5, S.FLUID, S.AIR)
    return np.round(8.0 * ONE * level).astype(np.int64), m, r


# ---- phi ----------------------------------------------------------------------------------------------------------------------
def test_phi_equals_an_independent_int64_evaluation():
    rng = np.random.default_rng(11)
    shape = (7, 6, 9)
    m = rng.integers(-1, 2, shape).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    m[2:4, 2:4, 2:4] = S.SOLID  # an obstacle: SOLID cells whose nearest non-SOLID cells are edge or vertex neighbours
    splat = rng.integers(0, 20 * ONE, shape).astype(np.int64)
    psi = S.wall_rule(splat, m)
    phi = S.smooth(psi)
    nz, ny, nx = shape

    def mk(z, y, x):
        return int(m[z, y, x]) if 0 <= z < nz and 0 <= y < ny and 0 <= x < nx else S.SOLID

    def comp(z, y, x):
        v = int(splat[z, y, x]) % 2 ** 64 >> 8
        return v + (9 << 28) * sum(mk(z + a, y + b, x + c) == S.SOLID for a, b, c in S.FACES)

    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                if mk(z, y, x) != S.SOLID:
                    want = comp(z, y, x)
                else:
                    want = 0
                    for shell in (1, 2, 3):
                        vals = [comp(z + a, y + b, x + c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)
                                if a * a + b * b + c * c == shell and mk(z + a, y + b, x + c) != S.SOLID]
                        if vals:
                            want = max(vals)
                            break
                assert psi[z, y, x] == want, (z, y, x)
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                want = sum((2 - a * a) * (2 - b * b) * (2 - c * c) * int(psi[min(max(z + a, 0), nz - 1), min(max(y + b, 0), ny - 1), min(max(x + c, 0), nx - 1)])
                           for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1))
                assert phi[z, y, x] == want, (z, y, x)


def test_phi_cannot_overflow_whatever_the_splat_holds():
    shape = (6, 6, 6)
    m = tank(shape)
    m[2:4, 2:4, 2:4] = S.FLUID
    splat = np.full(shape, -1, dtype=np.int64)  # 2^64 - 1 as the unsigned accumulator: above any sum of 2^32 particles' weights
    phi = S.smooth(S.wall_rule(splat, m))
    bound = 64 * ((2 ** 64 - 1 >> 8) + 6 * (9 << 28))
    assert bound < 2 ** 63
    assert int(phi.max()) <= bound and int(phi.min()) >= 0


# ---- curvature ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_a_pool_surface_against_the_walls_has_zero_curvature(axis):
    """A level surface along every axis, meeting the tank's SOLID walls: the splat near a wall lacks what the wall compensation adds back, as
    for particles that cannot sit in the wall."""
    shape = (14, 16, 12)
    m = tank(shape)
    idx = np.indices(shape)[axis]
    n = shape[axis]
    level = np.clip(0.6 * n - idx, 0.0, 1.0) * 8.0
    m[1:-1, 1:-1, 1:-1] = np.where(idx[1:-1, 1:-1, 1:-1] < int(0.6 * n), S.FLUID, S.AIR)
    nsolid = sum((S.shifted(m, *d, S.SOLID) == S.SOLID).astype(np.int64) for d in S.FACES)
    splat = (np.round(level * ONE).astype(np.int64) + (3 << 40) - ((9 << 28) << 8) * nsolid).astype(np.int64)
    phi, kappa = S.surface_field(splat, m)
    b = S.band(m)
    assert b.sum() > 0
    assert np.all(kappa == 0.0)


def test_a_tilted_plane_has_zero_curvature():
    shape = (16, 16, 16)
    m = tank(shape)
    z, y, x = np.indices(shape)
    m[1:-1, 1:-1, 1:-1] = np.where((x + 2 * y + 3 * z)[1:-1, 1:-1, 1:-1] < 45, S.FLUID, S.AIR)
    phi = ((1000 - (x + 2 * y + 3 * z)) * ONE).astype(np.int64)  # linear: every second difference is 0
    b = S.band(m)
    inner = np.zeros(shape, dtype=bool)
    inner[2:-2, 2:-2, 2:-2] = True
    k, zero = S.curvature64(phi, b & inner)
    assert (b & inner).sum() > 50
    assert np.all(k[b & inner] == 0.0) and not zero[b & inner].any()


@pytest.mark.parametrize("radius", [6, 10, 16])
def test_a_sphere_has_curvature_two_over_r_in_the_band(radius):
    n = 2 * radius + 12
    splat, m, r = radial_splat((n, n, n), (n / 2, n / 2, n / 2), radius)
    _, kappa = S.surface_field(splat, m)
    b = S.band(m)
    rel = np.abs(kappa[b] / (2.0 / r[b]) - 1.0)
    print(f"sphere R={radius}: {b.sum()} band cells, max relative error {rel.max():.4f}, mean {rel.mean():.4f}")
    assert rel.max() < 0.03


@pytest.mark.parametrize("radius", [6, 10])
def test_a_cylinder_has_curvature_one_over_r(radius):
    n = 2 * radius + 12
    splat, m, r = radial_splat((12, n, n), (0.0, n / 2, n / 2), radius, kind="cylinder")
    _, kappa = S.surface_field(splat, m)
    b = S.band(m)
    b[:4], b[-4:] = False, False  # the cells whose stencil reaches the compensated cells next to the z walls
    rel = np.abs(kappa[b] / (1.0 / r[b]) - 1.0)
    print(f"cylinder R={radius}: max relative error {rel.max():.4f}")
    assert rel.max() < 0.03


def test_a_bubble_has_negative_curvature():
    n = 32
    splat, m, r = radial_splat((n, n, n), (n / 2, n / 2, n / 2), 8, inside=False)
    _, kappa = S.surface_field(splat, m)
    b = S.band(m)
    assert np.all(kappa[b] < 0.0)
    assert np.abs(kappa[b] / (-2.0 / r[b]) - 1.0).max() < 0.03


def particle_sphere(radius, margin=6):
    """The splat and marker of an ideal drop: 8 particles per cell on the stratified lattice (cell + 0.25 / 0.75 per axis) inside a sphere of
    `radius`, splatted as the density scatter does (tent weights to the cell centres around the dual cell floor(p - 0.5)), FLUID where a
    particle sits."""
    n = int(2 * radius + 2 * margin)
    c = n / 2.0
    g = (np.arange(n)[:, None] + np.array([0.25, 0.75])[None, :]).ravel()
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    keep = (x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2 < radius ** 2
    pos = np.stack([x[keep], y[keep], z[keep]], axis=1)
    splat = np.zeros((n, n, n))
    d = np.floor(pos - 0.5).astype(int)
    for corner in range(8):
        o = np.array([corner & 1, (corner >> 1) & 1, corner >> 2])
        w = np.prod(np.clip(1.0 - np.abs(d + o + 0.5 - pos), 0.0, 1.0), axis=1)
        np.add.at(splat, (d[:, 2] + o[2], d[:, 1] + o[1], d[:, 0] + o[0]), w)
    m = tank((n, n, n))
    cell = np.floor(pos).astype(int)
    m[cell[:, 2], cell[:, 1], cell[:, 0]] = S.FLUID
    return np.round(splat * ONE).astype(np.int64), m


@pytest.mark.parametrize("radius, ratio", [(8, 0.7548), (12, 0.6680), (16, 0.5913)])
def test_the_curvature_of_a_splatted_drop_is_biased_low_and_more_so_for_larger_drops(radius, ratio):
    """The curvature the stage-1 rule measures on a realistic splat, pinned as a baseline: the mean over the FLUID-AIR faces of (k_i + k_j) / 2,
    the value the ghost faces carry, against 2/R.  The splat's surface profile is about two cells wide; on it the 3^3 central-difference
    formula is biased low, the more so the larger the drop, while on a wide ramp (the sphere test above) it is within 1 %.  This is the bias
    behind the low Laplace pressures and the long oscillation period measured on the GPU (DESIGN.md §8 "Surface tension"); a better
    curvature estimator must raise these ratios towards 1."""
    splat, m = particle_sphere(radius)
    _, kappa = S.surface_field(splat, m)
    faces = []
    for d in S.FACES:
        air = (m == S.FLUID) & (S.shifted(m, *d, S.SOLID) == S.AIR)
        faces.append((0.5 * (kappa.astype(np.float64) + S.shifted(kappa, *d, 0.0)))[air])
    mean = float(np.concatenate(faces).mean())
    print(f"splatted drop R={radius}: mean ghost-face curvature {mean / (2.0 / radius):.4f} of 2/R")
    assert abs(mean / (2.0 / radius) - ratio) <= 0.002


def test_curvature_is_clamped_and_zero_off_the_band():
    shape = (10, 10, 10)
    m = tank(shape)
    m[5, 5, 5] = S.FLUID
    splat = np.zeros(shape, dtype=np.int64)
    splat[5, 5, 5] = 8 * ONE
    _, kappa = S.surface_field(splat, m)
    b = S.band(m)
    assert np.all(np.abs(kappa) <= 2.0) and np.all(kappa[~b] == 0.0)
    assert kappa[5, 5, 5] == 0.0  # a symmetric peak: the three integer differences are 0
    assert kappa[5, 5, 6] == 2.0  # a one-cell drop is clamped to the curvature of a sphere of one cell radius


# ---- the pressure jump -----------------------------------------------------------------------------------------------------------
def test_a_sphere_of_uniform_curvature_is_an_equilibrium():
    """p == g inside solves the corrected system, and the corrected projection leaves every face at rest."""
    n, radius, dt, sigma = 20, 6, 1.0 / 120.0, 72.8
    _, m, _ = radial_splat((n, n, n), (n / 2, n / 2, n / 2), radius)
    kappa = np.where(S.band(m), np.float32(2.0 / radius), np.float32(0.0)).astype(np.float32)
    g = S.ghost(S.ghost_scale(dt, sigma), kappa.max(), kappa.max())
    rhs = S.rhs_after(np.zeros(m.shape, np.float32), m, kappa, dt, sigma)
    runs = pcg_ref.cg64(m, rhs, np.zeros(m.shape), 300)
    p = runs[-1][0]
    fl = m == S.FLUID
    # the float32 rhs holds n g rounded once per addition: the float64 solve lands within a few float32 roundings of g
    assert np.abs(p[fl] - float(g)).max() < 4e-6 * abs(float(g))
    p32 = np.where(fl, g, np.float32(0)).astype(np.float32)  # the equilibrium itself
    for axis in range(3):
        d = [(0, 0, 1), (0, 1, 0), (1, 0, 0)][axis]
        mn, pn = S.shifted(m, *d, S.SOLID), S.shifted(p32, *d, np.float32(0))
        live = (m != S.SOLID) & (mn != S.SOLID) & ((m == S.FLUID) | (mn == S.FLUID))
        u = np.where(live, (np.float32(0) - (p32 - pn)).astype(np.float32), np.float32(0))  # divergence_remove with p = 0 on AIR
        after = S.faces_after(u, m, kappa, dt, sigma, axis)
        assert np.all(after == 0.0), axis
        assert np.any(u != 0.0)  # without the correction the surface faces would move


def test_ghost_values_carry_the_sign_of_the_laplace_pressure():
    c = S.ghost_scale(1.0 / 120.0, 72.8)
    assert S.ghost(c, 0.25, 0.25) < 0.0 < S.ghost(c, -0.25, -0.25)  # p = -P dt / density: a drop's positive pressure is a negative p


# ---- capillary step limit -------------------------------------------------------------------------------------------------------
def test_capillary_limit_of_water_at_one_centimetre():
    assert S.capillary_limit_ns(72.8) == 33_062_018 > 8_333_333  # 33 ms: the default 1/120 s step is not cut


@pytest.mark.parametrize("sigma", [1e-3, 0.5, 72.8, 1e4, 1e8])
def test_capillary_limit_against_the_restatement(sigma):
    cap = S.capillary_limit_ns(sigma)
    assert cap == int(np.floor(1e9 * np.sqrt(1.0 / (4.0 * np.pi * float(np.float32(sigma))))))
    # plan_substep hands cfl_substep_ns the capped max_dt_ns: a quiet fluid takes the capillary limit (or the interval)
    assert cfl_ref.substep_ns(10 ** 12, [0.0, 0.0, 0.0], [0.0, 0.0, 0.0], 1.0, min(10 ** 12, cap), 1) == min(10 ** 12, cap)


def test_capillary_limit_falls_as_one_over_the_square_root_of_sigma():
    assert S.capillary_limit_ns(1e8) == 28_209
    for s in (1.0, 50.0, 3e3):
        assert abs(S.capillary_limit_ns(4.0 * s) - S.capillary_limit_ns(s) / 2.0) <= 1.0


# ---- scene key ------------------------------------------------------------------------------------------------------------------
def scene_with(tmp_path, value, scale=0.01):
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"]["grid_to_world_scale"] = scale
    if value is not None:
        sc["fluid"]["surface_tension"] = value
    p = tmp_path / "capillary.json"
    p.write_text(json.dumps(sc))
    return str(p)


def test_scene_surface_tension_is_converted_to_cells(tmp_path):
    assert F.scene_surface_tension(util.scene_path("dam_small")) == 0.0
    path = util.scene_path("droplet_zero_g")
    sc = json.load(open(path))
    s = np.float32(sc["fluid"]["grid_to_world_scale"])
    assert F.scene_surface_tension(path) == float(np.float32(sc["fluid"]["surface_tension"]) / (s * s * s)) > 0.0
    water = F.scene_surface_tension(scene_with(tmp_path, 7.28e-5, 0.01))
    assert water == float(np.float32(7.28e-5) / (np.float32(0.01) * np.float32(0.01) * np.float32(0.01)))
    assert abs(water - 72.8) < 1e-3
    assert F.scene_surface_tension(scene_with(tmp_path, None)) == 0.0
    assert blub_b200.scene_info(scene_with(tmp_path, 0)).max_num_particles > 0


@pytest.mark.parametrize("value", [-1e-5, "wet", [1.0], {"x": 1}, 1e39, True, None])
def test_scene_surface_tension_refuses_bad_values(tmp_path, value):
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"]["surface_tension"] = value
    p = tmp_path / "bad.json"
    p.write_text(json.dumps(sc))
    L = F.lib()
    assert L.blub_scene_info(os.fsencode(str(p)), F.SceneInfo()) == BLUB_ERR_PARSE
    assert L.blub_scene_surface_tension(os.fsencode(str(p)), F.C.c_float()) == BLUB_ERR_PARSE


def test_scene_surface_tension_overflowing_in_cells_is_refused(tmp_path):
    L = F.lib()
    assert L.blub_scene_surface_tension(os.fsencode(scene_with(tmp_path, 1e30, 1e-4)), F.C.c_float()) == BLUB_ERR_PARSE


# ---- state file version 64 ------------------------------------------------------------------------------------------------------
def st_payload(sigma=72.8, reserved=0):
    return struct.pack("<fI", sigma, reserved)


def promote64(base, num_sections, viscous=False, payload=None, tail=b"", corrupt_crc=False, version=64):
    """A file of an older version with its header rewritten to `version` and `num_sections`, section 17 (when viscous) and 18 behind it."""
    data = bytearray(base)
    data[8:12] = struct.pack("<I", version)
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", num_sections)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    payload = st_payload() if payload is None else payload
    sec = section(18, payload)
    if corrupt_crc:
        sec = sec[:-4] + struct.pack("<I", zlib.crc32(payload) ^ 1)
    return bytes(data) + (section(17, viscosity_payload()) if viscous else b"") + sec + tail


BASES = {
    "13 sections": (lambda: state_bytes(), 13),
    "flow section": (lambda: state_bytes() + section(14, bytes(1056)), 14),
    "bodies": (lambda: v8_bytes(BODIES), 15),
    "mesh body": (lambda: v16_bytes(), 16),
}


@pytest.mark.parametrize("viscous", [False, True])
@pytest.mark.parametrize("base", sorted(BASES))
def test_version_64_written_from_the_documented_layout_is_accepted(tmp_path, base, viscous):
    make, nb = BASES[base]
    info = F.state_info(write(tmp_path, promote64(make(), nb + 1 + viscous, viscous)))
    assert info.format_version == 64


@pytest.mark.parametrize("case, make, needle", [
    ("surface tension 0", lambda: promote64(state_bytes(), 14, payload=st_payload(0.0)), "above 0"),
    ("surface tension NaN", lambda: promote64(state_bytes(), 14, payload=st_payload(float("nan"))), "above 0"),
    ("surface tension negative", lambda: promote64(v8_bytes(BODIES), 16, payload=st_payload(-1.0)), "above 0"),
    ("reserved", lambda: promote64(state_bytes(), 14, payload=st_payload(reserved=1)), "reserved"),
    ("section 18 too long", lambda: promote64(state_bytes(), 14, payload=st_payload() + bytes(4)), "its header describes"),
    ("section 18 too short", lambda: promote64(state_bytes(), 14, payload=st_payload()[:4]), "its header describes"),
    ("num_sections names another layout", lambda: promote64(state_bytes(), 15), "its header describes"),
    ("num_sections names no layout", lambda: promote64(state_bytes(), 13), "14 to 17"),
    ("viscous, num_sections names no layout", lambda: promote64(state_bytes(), 14, viscous=True), "15 to 18"),
    ("trailing bytes", lambda: promote64(state_bytes(), 14, tail=bytes(4)), "its header describes"),
    ("bad CRC", lambda: promote64(state_bytes(), 14, corrupt_crc=True), "checksum mismatch in section 18"),
    ("viscosity 0 in section 17", lambda: promote64(state_bytes(), 15, viscous=True)[:-(20 + 8 + 36)] + section(17, viscosity_payload(nu=0.0))
     + section(18, st_payload()), "above 0"),
] + [(f"version {v}", (lambda v=v: promote64(state_bytes(), 14, version=v)), "version") for v in (33, 48, 63, 65, 128)])
def test_malformed_version_64_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    assert rc == BLUB_ERR_PARSE, (case, rc)
    assert needle in L.blub_last_error().decode(), (case, L.blub_last_error().decode())
