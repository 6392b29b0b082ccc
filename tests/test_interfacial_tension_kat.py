"""CPU: known answers of the interfacial tension rule (DESIGN.md §8 "Interfacial tension") through its NumPy restatement
tests/interfacial_tension_ref.py: the phase field against Python integers, the curvature of analytic interfaces, the exact equilibrium of a
drop with and without a density table, the capillary limit, the scene key and the version-512 state file as the host-only reader sees it.
No GPU needed."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import interfacial_tension_ref as I, pcg_ref, surface_tension_ref as S, tag_density_ref as T, util
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes, write
from tests.test_tag_viscosity_kat import V256_BASES, st_payload, td_payload, tv_payload
from tests.test_viscosity_kat import viscosity_payload

BLUB_ERR_PARSE = 5
ONE = 1 << 40  # one particle weight in the splat's fixed point


def tank(shape, fill=I.FLUID):
    m = np.full(shape, fill, dtype=np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


# ---- psi and phi ----------------------------------------------------------------------------------------------------------------
def test_phi_equals_an_independent_python_integer_evaluation():
    rng = np.random.default_rng(5)
    shape = (7, 6, 9)
    m = rng.integers(-1, 2, shape).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    m[2:4, 2:4, 2:4] = I.SOLID  # an obstacle: SOLID cells whose nearest non-SOLID cells are edge or vertex neighbours
    splat_all = rng.integers(0, 20 * ONE, shape).astype(np.int64)
    splat_b = (splat_all * rng.random(shape)).astype(np.int64)
    splat_b[1, 1, 1] = splat_all[1, 1, 1] // 2  # psi == 0 up to the borrow
    phi = I.phase_field(splat_all, splat_b, m)
    nz, ny, nx = shape

    def mk(z, y, x):
        return int(m[z, y, x]) if 0 <= z < nz and 0 <= y < ny and 0 <= x < nx else I.SOLID

    def comp(z, y, x):
        v = (2 * int(splat_b[z, y, x]) - int(splat_all[z, y, x])) >> 8  # Python integers: exact, floor shift
        sign = (v > 0) - (v < 0)
        return v + sign * (9 << 28) * sum(mk(z + a, y + b, x + c) == I.SOLID for a, b, c in I.FACES)

    psi = {}
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                if m[z, y, x] != I.SOLID:
                    psi[z, y, x] = comp(z, y, x)
                    continue
                v = 0
                for shell in (1, 2, 3):
                    cand = [comp(z + c, y + b, x + a) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)
                            if a * a + b * b + c * c == shell and mk(z + c, y + b, x + a) != I.SOLID]
                    if cand:
                        v = max(cand, key=lambda t: (abs(t), t))
                        break
                psi[z, y, x] = v
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                want = sum((2 - a * a) * (2 - b * b) * (2 - c * c) * psi[min(max(z + c, 0), nz - 1), min(max(y + b, 0), ny - 1), min(max(x + a, 0), nx - 1)]
                           for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1))
                assert int(phi[z, y, x]) == want, (z, y, x)


def test_phi_cannot_overflow_whatever_the_splats_hold():
    shape = (6, 6, 6)
    m = tank(shape)
    m[2:4, 2:4, 2:4] = I.SOLID
    top = np.full(shape, -1, dtype=np.int64)  # 2^64 - 1 as unsigned
    for splat_all, splat_b in ((top, np.zeros(shape, np.int64)), (np.zeros(shape, np.int64), top), (top, top)):
        phi = I.phase_field(splat_all, splat_b, m)
        bound = 64 * ((1 << 56) + 6 * (9 << 28))
        assert bound < 2 ** 63
        assert int(np.abs(phi).max()) <= bound


# ---- curvature of analytic interfaces ---------------------------------------------------------------------------------------------
def radial_splats(shape, centre, radius, kind="sphere", inside=True, width=8.0):
    """8 particle weights per cell everywhere; phase B a sphere (or a cylinder along z) with a linear ramp of `width` cells, its complement
    when not `inside`.  The marker is FLUID inside the tank."""
    z, y, x = np.indices(shape, dtype=np.float64) + 0.5
    d2 = (x - centre[2]) ** 2 + (y - centre[1]) ** 2 + (0.0 if kind == "cylinder" else (z - centre[0]) ** 2)
    r = np.sqrt(d2)
    level = np.clip(0.5 - (r - radius) / width, 0.0, 1.0)
    if not inside:
        level = 1.0 - level
    splat_all = np.full(shape, 8 * ONE, dtype=np.int64)
    return splat_all, np.round(8.0 * ONE * level).astype(np.int64), tank(shape), r


@pytest.mark.parametrize("radius", [6, 10])
def test_a_drop_of_b_has_curvature_two_over_r(radius):
    n = 2 * radius + 12
    sa, sb, m, r = radial_splats((n, n, n), (n / 2, n / 2, n / 2), radius)
    phi, kappa = I.interface_field(sa, sb, m)
    b = I.band(phi, m)
    assert b.sum() > 50
    assert np.abs(kappa[b] / (2.0 / r[b]) - 1.0).max() < 0.03
    assert not kappa[~b].any()


@pytest.mark.parametrize("radius", [6, 10])
def test_a_cylinder_of_b_has_curvature_one_over_r(radius):
    n = 2 * radius + 12
    sa, sb, m, r = radial_splats((16, n, n), (0.0, n / 2, n / 2), radius, kind="cylinder")
    phi, kappa = I.interface_field(sa, sb, m)
    # away from the end walls: this synthetic splat is not thinned next to a wall as a particle splat is, so the wall compensation, which
    # changes sign across the interface, would add a step there (the layer tests below meet the walls with splats that are)
    b = I.band(phi, m)
    b[:4], b[12:] = False, False
    assert np.abs(kappa[b] / (1.0 / r[b]) - 1.0).max() < 0.03


def test_a_drop_of_a_in_b_has_the_opposite_sign():
    n = 32
    sa, sb, m, r = radial_splats((n, n, n), (n / 2, n / 2, n / 2), 8, inside=False)
    phi, kappa = I.interface_field(sa, sb, m)
    b = I.band(phi, m)
    assert np.all(kappa[b] < 0.0)
    assert np.abs(kappa[b] / (-2.0 / r[b]) - 1.0).max() < 0.03


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_flat_layers_meeting_the_tank_walls_have_zero_curvature(axis):
    """Phase B below a level along every axis, across the whole tank: the walls' signed compensation mirrors both phases."""
    shape = (14, 16, 12)
    m = tank(shape)
    coord = np.indices(shape)[axis]
    half = shape[axis] // 2
    # particles cannot sit in the wall cells: a cell loses 0.5625 particle weights of its splat per SOLID face neighbour
    nsolid = sum((S.shifted(m, *d, I.SOLID) == I.SOLID).astype(np.int64) for d in I.FACES)
    sa = np.where(m != I.SOLID, 8 * ONE - (9 << 36) * nsolid, 0).astype(np.int64)
    sb = np.where(coord < half, sa, 0).astype(np.int64)
    phi, kappa = I.interface_field(sa, sb, m)
    b = I.band(phi, m)
    assert b.sum() == 2 * np.prod([s - 2 for k, s in enumerate(shape) if k != axis])
    assert not kappa.any()


def lattice_drop(radius, margin=5, wall_layer=None):
    """Every cell inside the tank holds 8 particles on the stratified lattice, splatted as the density scatter does; phase B a sphere of
    `radius` (or, with wall_layer = h, the layer y < h)."""
    n = int(2 * radius + 2 * margin)
    c = n / 2.0
    g = (np.arange(1, n - 1)[:, None] + np.array([0.25, 0.75])[None, :]).ravel()
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    pos = np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1)
    if wall_layer is None:
        in_b = ((pos - c) ** 2).sum(axis=1) < radius ** 2
    else:
        in_b = pos[:, 1] < wall_layer
    sa, sb = np.zeros((n, n, n)), np.zeros((n, n, n))
    d = np.floor(pos - 0.5).astype(int)
    for corner in range(8):
        o = np.array([corner & 1, (corner >> 1) & 1, corner >> 2])
        w = np.prod(np.clip(1.0 - np.abs(d + o + 0.5 - pos), 0.0, 1.0), axis=1)
        idx = (d[:, 2] + o[2], d[:, 1] + o[1], d[:, 0] + o[0])
        np.add.at(sa, idx, w)
        np.add.at(sb, tuple(i[in_b] for i in idx), w[in_b])
    return np.round(sa * ONE).astype(np.int64), np.round(sb * ONE).astype(np.int64), tank((n, n, n))


@pytest.mark.parametrize("radius, ratio", [(8, 1.0350), (12, 1.0725)])
def test_the_curvature_of_a_splatted_b_drop_is_pinned(radius, ratio):
    """The mean of (k_i + k_j) / 2 over the interface faces of a lattice drop against 2/R, pinned as a baseline.  Unlike the free surface's
    (0.75 / 0.67 of 2/R, tests/test_surface_tension_kat.py) it is not biased low: phi runs from -8 to +8 particle weights across the
    interface, twice the free surface's rise, and the faces sit where phi changes sign, in the middle of the profile."""
    sa, sb, m = lattice_drop(radius)
    phi, kappa = I.interface_field(sa, sb, m)
    vals = [(0.5 * (kappa.astype(np.float64) + S.shifted(kappa, *d, 0.0)))[mask] for d, mask in I.interface_faces(phi, m)]
    mean = float(np.concatenate(vals).mean())
    print(f"splatted B drop R={radius}: mean interface curvature {mean / (2.0 / radius):.4f} of 2/R")
    assert abs(mean / (2.0 / radius) - ratio) <= 0.002


def test_a_splatted_flat_layer_at_the_walls_is_flat_away_from_the_walls():
    """A lattice layer y < 8 across the whole tank: zero curvature on the interface except within 3 cells of a side wall, where the wall
    compensation, whose sign follows the cell's phase, restores one phase's missing weight but not the other's; the largest value is pinned
    (0.0143, a radius of 70 cells)."""
    sa, sb, m = lattice_drop(6, wall_layer=8.0)
    phi, kappa = I.interface_field(sa, sb, m)
    b = I.band(phi, m)
    assert b.sum() > 100
    n = m.shape[0]
    z, y, x = np.indices(m.shape)
    wall_distance = np.minimum(np.minimum(x, n - 1 - x), np.minimum(z, n - 1 - z))
    assert not kappa[wall_distance > 3].any()  # the smoothing carries the wall cells' error three cells in
    print(f"flat layer: max |kappa| within 3 cells of a side wall {np.abs(kappa).max():.4f}")
    assert np.abs(kappa).max() <= 0.0144


# ---- the pressure jump --------------------------------------------------------------------------------------------------------------
def drop_scene(n=20, radius=6):
    """A B sphere of uniform band curvature 2/R in A, with AIR above y = n - 4 so that the solve has a Dirichlet boundary."""
    m = tank((n, n, n))
    m[:, n - 4:-1, :] = I.AIR
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    z, y, x = np.indices(m.shape) + 0.5
    inside = (x - n / 2) ** 2 + (y - n / 2 + 3) ** 2 + (z - n / 2) ** 2 < radius ** 2
    phi = np.where(inside, 1, -1).astype(np.int64)
    kappa = np.where(I.band(phi, m), np.float32(2.0 / radius), np.float32(0)).astype(np.float32)
    return m, phi, kappa


@pytest.mark.parametrize("table", [False, True])
def test_a_drop_of_uniform_curvature_is_an_exact_equilibrium(table):
    """p = g on B and 0 on A solves the corrected system; the corrected projection leaves every face at rest; the float64 solve finds it."""
    m, phi, kappa = drop_scene()
    dt, s = 1.0 / 120.0, 200.0
    g = S.ghost(S.ghost_scale(dt, s), kappa.max(), kappa.max())
    fl = m == I.FLUID
    b = I.phase_b(phi, m)
    if table:
        rho = np.where(fl, np.where(b, np.float32(0.8), np.float32(1.0)), np.float32(0)).astype(np.float32)
        beta, D, _ = T.coefficients(m, rho)
    else:
        beta = None
    rhs = I.rhs_after(np.zeros(m.shape, np.float32), m, phi, kappa, dt, s, beta)
    assert np.count_nonzero(rhs) > 100
    if table:
        A, idx = T.matrix(beta, D, fl)
        p = np.zeros(m.shape)
        p[fl] = T.solve64(A, rhs.astype(np.float64)[fl])
    else:
        p = pcg_ref.cg64(m, rhs, np.zeros(m.shape), 400)[-1][0]
    # the float32 rhs holds up to six weighted g rounded once per addition: the float64 solve lands within a few float32 roundings
    assert np.abs(p[b] - float(g)).max() < 2e-5 * abs(float(g))
    assert np.abs(p[fl & ~b]).max() < 2e-5 * abs(float(g))
    p32 = np.where(b, g, np.float32(0)).astype(np.float32)  # the equilibrium itself
    for axis in range(3):
        d = [(0, 0, 1), (0, 1, 0), (1, 0, 0)][axis]
        mn, pn = S.shifted(m, *d, I.SOLID), S.shifted(p32, *d, np.float32(0))
        live = (m != I.SOLID) & (mn != I.SOLID) & ((m == I.FLUID) | (mn == I.FLUID))
        if table:
            du = (beta[axis] * (p32 - pn)).astype(np.float32)
        else:
            du = (p32 - pn).astype(np.float32)
        u = np.where(live, (np.float32(0) - du).astype(np.float32), np.float32(0))  # divergence_remove
        after = I.faces_after(u, m, phi, kappa, dt, s, axis, beta)
        assert np.all(after == 0.0), axis
        assert np.any(u != 0.0)  # without the correction the interface faces would move


def test_a_drop_of_b_carries_a_positive_laplace_pressure():
    c = S.ghost_scale(1.0 / 120.0, 200.0)
    assert S.ghost(c, 0.25, 0.25) < 0.0  # p = -P dt / density: P_B - P_A = s kappa > 0 for a B drop is a negative p jump


# ---- capillary limit and scene key --------------------------------------------------------------------------------------------------
def test_capillary_limit_takes_the_larger_tension():
    assert I.capillary_limit_ns(0.0, 200.0) == S.capillary_limit_ns(200.0)
    assert I.capillary_limit_ns(72.8, 200.0) == S.capillary_limit_ns(200.0)
    assert I.capillary_limit_ns(300.0, 200.0) == S.capillary_limit_ns(300.0)


def scene_with(tmp_path, value):
    sc = json.load(open(util.scene_path("oil_water_small")))
    sc["fluid"]["interfacial_tension"] = value
    p = tmp_path / "it.json"
    p.write_text(json.dumps(sc))
    return str(p)


def test_scene_interfacial_tension_is_converted_to_cells(tmp_path):
    assert F.scene_interfacial_tension(util.scene_path("dam_small")) == (0.0, [])
    s, tags = F.scene_interfacial_tension(scene_with(tmp_path, {"tags": [1, 7], "tension": 3e-5}))
    assert tags == [1, 7]
    assert s == pytest.approx(3e-5 / 0.01 ** 3, rel=1e-6)
    s, tags = F.scene_interfacial_tension(util.scene_path("oil_drop_zero_g"))
    assert tags == [1] and s > 0.0


@pytest.mark.parametrize("value", [
    {"tags": [1], "tension": -1e-5}, {"tags": [1], "tension": "x"}, {"tags": [], "tension": 1e-5}, {"tags": [1, 1], "tension": 1e-5},
    {"tags": list(range(17)), "tension": 1e-5}, {"tension": 1e-5}, {"tags": [1]}, [1, 2], 3e-5, {"tags": [1], "tension": 1e35},
    {"tags": [-1], "tension": 1e-5}])
def test_scene_interfacial_tension_refuses_bad_values(tmp_path, value):
    path = os.fsencode(scene_with(tmp_path, value))
    L = F.lib()
    count, s = F.C.c_uint32(0), F.C.c_float(0)
    assert L.blub_scene_interfacial_tension(path, None, 0, F.C.byref(count), F.C.byref(s)) == BLUB_ERR_PARSE
    assert L.blub_scene_surface_tension(path, F.C.byref(s)) == BLUB_ERR_PARSE  # every scene call


def test_a_zero_tension_in_a_scene_is_accepted_without_tags(tmp_path):
    assert F.scene_interfacial_tension(scene_with(tmp_path, {"tags": [], "tension": 0.0})) == (0.0, [])


# ---- state format version 512 ---------------------------------------------------------------------------------------------------------
def it_payload(tension=200.0, tags=(1,), count=None, tail=()):
    rows = list(tags) + list(tail)
    return struct.pack("<fI", tension, len(tags) if count is None else count) + struct.pack(f"<{len(rows)}I", *rows) + bytes(4 * (16 - len(rows)))


def promote512(base, nb, s17=None, with18=False, with19=False, s20=None, payload=None, version=512, with21=True):
    """A base layout of nb sections rewritten to `version`, then the setting sections asked for in the order 17, 18, 19, 20, and 21."""
    data = bytearray(base)
    ns = nb + (s17 is not None) + with18 + with19 + (s20 is not None) + with21
    data[8:12] = struct.pack("<I", version)
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", ns)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    out = bytes(data)
    if s17 is not None:
        out += section(17, s17)
    if with18:
        out += section(18, st_payload())
    if with19:
        out += section(19, td_payload())
    if s20 is not None:
        out += section(20, s20)
    return out + (section(21, it_payload() if payload is None else payload) if with21 else b"")


# the setting sections a fluid can write before section 21: 18 and 19 are exclusive, 20 comes with 17, 19 not with floating bodies
EXTRAS = {"none": {}, "17": {"s17": viscosity_payload(nu=3.0)}, "18": {"with18": True}, "19": {"with19": True},
          "17+20": {"s17": viscosity_payload(nu=0.0), "s20": tv_payload()}, "17+18+20": {"s17": viscosity_payload(nu=3.0), "with18": True, "s20": tv_payload()},
          "17+19+20": {"s17": viscosity_payload(nu=0.0), "with19": True, "s20": tv_payload()}}


@pytest.mark.parametrize("base,extra", [(b, e) for b in sorted(V256_BASES) for e in sorted(EXTRAS)
                                        if not ("19" in e and b in ("bodies", "mesh body"))])
def test_version_512_written_from_the_documented_layout_is_accepted(tmp_path, base, extra):
    make, nb = V256_BASES[base]
    info = F.state_info(write(tmp_path, promote512(make(), nb, **EXTRAS[extra])))
    assert info.format_version == 512


def parse_error(tmp_path, data):
    path = write(tmp_path, data)
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    return rc, L.blub_last_error().decode()


@pytest.mark.parametrize("case, make, needle", [
    ("no section 21", lambda: promote512(state_bytes(), 13, with21=False, s17=viscosity_payload(nu=3.0)), "version"),
    ("version-256 layout", lambda: promote512(state_bytes(), 13, s17=viscosity_payload(nu=3.0), s20=tv_payload(), with21=False), "version"),
    ("truncated section 21", lambda: promote512(state_bytes(), 13, payload=it_payload()[:-8]), "its header describes"),
    ("tension 0", lambda: promote512(state_bytes(), 13, payload=it_payload(tension=0.0)), "above 0"),
    ("tension NaN", lambda: promote512(state_bytes(), 13, payload=it_payload(tension=float("nan"))), "section 21"),
    ("tension negative", lambda: promote512(state_bytes(), 13, payload=it_payload(tension=-1.0)), "section 21"),
    ("no tags", lambda: promote512(state_bytes(), 13, payload=it_payload(tags=())), "section 21"),
    ("count above 16", lambda: promote512(state_bytes(), 13, payload=it_payload(count=17)), "1 to 16"),
    ("duplicate tag", lambda: promote512(state_bytes(), 13, payload=it_payload(tags=(1, 1))), "twice"),
    ("unused entry not zero", lambda: promote512(state_bytes(), 13, payload=it_payload(tail=(5,))), "unused"),
    ("section 17 zero without 20", lambda: promote512(state_bytes(), 13, s17=viscosity_payload(nu=0.0)), "above 0"),
    ("section 20 without 17", lambda: promote512(state_bytes(), 13, s20=tv_payload()), "section 17"),
    ("sections 18 and 19 together", lambda: promote512(state_bytes(), 13, with18=True, with19=True), "surface tension"),
    ("section 19 with bodies", lambda: promote512(v8_bytes(BODIES), 15, with19=True), "floating bodies"),
] + [(f"version {v}", (lambda v=v: promote512(state_bytes(), 13, version=v)), "version") for v in (257, 300, 511, 513, 1024)])
def test_malformed_version_512_files_are_parse_errors(tmp_path, case, make, needle):
    rc, msg = parse_error(tmp_path, make())
    assert rc == BLUB_ERR_PARSE, (case, rc, msg)
    assert needle in msg, (case, msg)
