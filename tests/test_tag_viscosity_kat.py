"""Known-answer tests of the tag viscosity restatement (tests/tag_viscosity_ref.py) and of the scene key: the per-pair system is symmetric
with smallest eigenvalue >= 1, every live face's pair sets are non-empty, a uniform table is visc_ref's matrix, an all-zero table makes no
unknowns, the cell viscosity does not depend on the particle order, and a two-layer Couette flow has the slope ratio nu_2 / nu_1."""
import json
import os
import struct
import zlib

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import blub_b200
from blub_b200 import fluid as F
from tests import tag_viscosity_ref as R, util, visc_ref as V
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_mesh_bodies_kat import v16_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes, write
from tests.test_surface_tension_kat import st_payload
from tests.test_tag_density_kat import td_payload
from tests.test_viscosity_kat import viscosity_payload

BLUB_ERR_PARSE = 5

DT32 = float(np.float32(1.0 / 120.0))


def salt_and_pepper(shape, seed):
    rng = np.random.default_rng(seed)
    m = rng.integers(-1, 2, shape).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def tagged_particles(marker, seed, per_cell=3, tags=(0, 1, 2)):
    """Particles in every FLUID cell (and a few in SOLID ones), random tags."""
    rng = np.random.default_rng(seed)
    z, y, x = np.nonzero(marker != AIR_)
    keep = (marker[z, y, x] == R.FLUID) | (rng.random(len(z)) < 0.1)
    z, y, x = z[keep], y[keep], x[keep]
    cells = np.repeat(np.stack([x, y, z], 1), per_cell, 0).astype(np.float32)
    pos = cells + rng.uniform(0.05, 0.95, cells.shape).astype(np.float32)
    return pos, rng.choice(np.array(tags, dtype=np.uint32), len(pos))


AIR_ = R.AIR


def systems(marker, table, fluid_nu, seed, vox=None):
    pos, tags = tagged_particles(marker, seed)
    nu = R.cell_viscosity(pos, tags, table, fluid_nu, marker)
    rng = np.random.default_rng(seed + 1)
    return [R.PairSystem(marker, c, nu, DT32, rng.standard_normal(marker.shape).astype(np.float32), 0.1 * c, vox) for c in range(3)], nu


@pytest.mark.parametrize("table,fluid_nu", [({1: 120.0, 2: 1.2}, 0.0), ({1: 1200.0}, 12.0), ({0: 0.0, 1: 60.0, 2: 6000.0}, 3.0)])
@pytest.mark.parametrize("solid", [False, True])
def test_matrix_is_symmetric_with_smallest_eigenvalue_at_least_one(table, fluid_nu, solid):
    marker = salt_and_pepper((10, 12, 14), 3)
    vox = None
    if solid:  # a moving solid: every voxel carries a velocity
        vox = np.random.default_rng(5).uniform(-2, 2, marker.shape + (4,)).astype(np.float16)
    ss, _ = systems(marker, table, fluid_nu, 7, vox)
    for c, s in enumerate(ss):
        assert R.pair_sets_nonempty(marker, c)
        assert s.n > 0
        A = s.A.toarray()
        assert np.array_equal(A, A.T)
        assert np.linalg.eigvalsh(A).min() >= 1.0 - 1e-12
        assert (np.asarray(s.A.diagonal()) - np.abs(A - np.diag(np.diag(A))).sum(1) >= 1.0 - 1e-12).all()  # strictly diagonally dominant


def test_uniform_table_is_the_constant_matrix():
    marker = salt_and_pepper((10, 12, 14), 4)
    nu = 90.0
    ss, nu_cells = systems(marker, {0: nu, 1: nu, 2: nu}, nu, 9)
    assert (nu_cells[marker == R.FLUID] == np.float32(nu)).all()
    k32 = float(np.float32(nu) * np.float32(DT32))
    for c, s in enumerate(ss):
        ref = V.System(marker, c, k32, np.zeros(marker.shape, np.float32), 0.0)
        assert np.array_equal(s.live, ref.live)
        assert abs(s.A - ref.A).max() == 0.0


def test_all_zero_table_makes_no_unknowns():
    marker = salt_and_pepper((10, 12, 14), 5)
    ss, nu = systems(marker, {0: 0.0, 1: 0.0, 2: 0.0}, 0.0, 11)
    assert not nu.any() and all(s.n == 0 for s in ss)


def test_cell_viscosity_does_not_depend_on_particle_order():
    marker = salt_and_pepper((10, 12, 14), 6)
    pos, tags = tagged_particles(marker, 13, per_cell=5)
    table = {0: 1.0, 1: 1000.0, 2: 1e-7}
    a = R.cell_viscosity(pos, tags, table, 3.0, marker)
    perm = np.random.default_rng(1).permutation(len(pos))
    b = R.cell_viscosity(pos[perm], tags[perm], table, 3.0, marker)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    # a value below nu_scale 2^-33 adds 0: tag 2 alone in a cell gives exactly 0
    assert R.q_of(1e-7, 1000.0) == 0


@pytest.mark.parametrize("ratio", [10.0, 100.0])
def test_two_layer_couette_slope_ratio(ratio):
    """Two layers between the floor at rest and a SOLID lid moving at U along x; AIR on the x and z sides makes every free-surface
    neighbour drop, so the problem is one-dimensional in y.  The steady state of the operator without its identity has a constant flux."""
    nx, ny, nz, U = 8, 22, 6, 1.0
    marker = np.full((nz, ny, nx), R.AIR, np.int8)
    marker[1:-1, 1:ny - 1, 2:-2] = R.FLUID  # two AIR columns on the x sides: no face reaches the grid's outside along x
    marker[:, 0, :] = R.SOLID
    marker[:, ny - 1, :] = R.SOLID
    vox = np.zeros((nz, ny, nx, 4), np.float16)
    vox[:, ny - 1, :, 0] = U
    nu1 = 10.0
    nu = np.where(marker == R.FLUID, np.float32(nu1), np.float32(0)).astype(np.float32)
    half = ny // 2
    nu[:, half:, :][marker[:, half:, :] == R.FLUID] = np.float32(nu1 * ratio)
    s = R.PairSystem(marker, 0, nu, DT32, np.zeros(marker.shape, np.float32), 0.0, vox)
    # steady state: solve (A - I) x = b - w without the identity (w = 0 here)
    A = (s.A - sp.eye(s.n)).tocsc()
    x = spl.spsolve(A, s.b)
    u = np.full(marker.shape, np.nan)
    u[s.live] = x
    col = u[nz // 2, 1:ny - 1, nx // 2]  # faces between x = nx/2 and nx/2 + 1 along y
    slopes = np.diff(col)
    low, high = slopes[2:half - 3], slopes[half + 1:-2]
    assert np.allclose(low, low[0], rtol=1e-9) and np.allclose(high, high[0], rtol=1e-9)
    # the flux k dx is constant: the slope ratio is that of the float32 coefficients, nu_2 / nu_1 to their rounding
    k1, k2 = float(np.float32(nu1) * np.float32(DT32)), float(np.float32(nu1 * ratio) * np.float32(DT32))
    assert abs(low[0] / high[0] / (k2 / k1) - 1.0) < 1e-9 and abs(k2 / k1 / ratio - 1.0) < 1e-6


# ---- scene key ------------------------------------------------------------------------------------------------------------------
def write_scene(tmp_path, entries):
    s = json.load(open(util.scene_path("honey_water_small")))
    if entries is None:
        del s["fluid"]["tag_viscosities"]
    else:
        s["fluid"]["tag_viscosities"] = entries
    p = tmp_path / "s.json"
    p.write_text(json.dumps(s))
    return str(p)


def test_scene_key_in_cells2_per_s(tmp_path):
    assert F.scene_tag_viscosities(util.scene_path("honey_water_small")) == {1: pytest.approx(0.01 / 1e-4, rel=1e-6)}
    assert F.scene_tag_viscosities(write_scene(tmp_path, None)) == {}
    assert F.scene_tag_viscosities(write_scene(tmp_path, [])) == {}


@pytest.mark.parametrize("entries", [
    {"tag": 1, "viscosity": 1.0},
    [1.0],
    [{"tag": 1}],
    [{"viscosity": 1.0}],
    [{"tag": 1, "viscosity": -1.0}],
    [{"tag": 1, "viscosity": "x"}],
    [{"tag": -1, "viscosity": 1.0}],
    [{"tag": 1, "viscosity": 1.0}, {"tag": 1, "viscosity": 2.0}],
    [{"tag": t, "viscosity": 1.0} for t in range(17)],
    [{"tag": 1, "viscosity": 1e38}],
])
def test_scene_key_parse_errors(tmp_path, entries):
    path = write_scene(tmp_path, entries)
    with pytest.raises(blub_b200.BlubError):
        F.scene_tag_viscosities(path)
    count = F.C.c_uint32(0)
    out = (F.TagViscosity * 16)()
    assert F.lib().blub_scene_tag_viscosities(os.fsencode(path), out, 16, F.C.byref(count)) == BLUB_ERR_PARSE
    assert F.lib().blub_scene_info(os.fsencode(path), F.SceneInfo()) == BLUB_ERR_PARSE


# ---- state format version 256 ---------------------------------------------------------------------------------------------------
def tv_payload(entries=((1, 100.0),), count=None, reserved=0, tail=()):
    out = struct.pack("<II", len(entries) if count is None else count, reserved)
    rows = list(entries) + list(tail)
    for tag, nu in rows:
        out += struct.pack("<If", tag, nu)
    return out + bytes(8 * (16 - len(rows)))


def promote256(base, nb, nu=0.0, with18=False, with19=False, payload=None, version=256, s17=None):
    """A base layout of nb sections rewritten to `version`, then section 17 (nu), 18 and 19 when asked, and 20."""
    data = bytearray(base)
    ns = nb + 2 + with18 + with19
    data[8:12] = struct.pack("<I", version)
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", ns)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    out = bytes(data) + section(17, viscosity_payload(nu=nu) if s17 is None else s17)
    if with18:
        out += section(18, st_payload())
    if with19:
        out += section(19, td_payload())
    return out + section(20, tv_payload() if payload is None else payload)


V256_BASES = {"13 sections": (lambda: state_bytes(), 13), "flow section": (lambda: state_bytes() + section(14, bytes(1056)), 14),
              "bodies": (lambda: v8_bytes(BODIES), 15), "mesh body": (lambda: v16_bytes(), 16)}


# section 19 only on the bases without floating bodies, which a tag density table does not support
@pytest.mark.parametrize("base,extra", [(b, e) for b in sorted(V256_BASES) for e in ("none", "18", "19")
                                        if not (e == "19" and b in ("bodies", "mesh body"))])
@pytest.mark.parametrize("nu", [0.0, 3.0])
def test_version_256_written_from_the_documented_layout_is_accepted(tmp_path, base, nu, extra):
    make, nb = V256_BASES[base]
    info = F.state_info(write(tmp_path, promote256(make(), nb, nu, extra == "18", extra == "19")))
    assert info.format_version == 256


def parse_error(tmp_path, data):
    path = write(tmp_path, data)
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    return rc, L.blub_last_error().decode()


@pytest.mark.parametrize("case, make, needle", [
    ("truncated section 20", lambda: promote256(state_bytes(), 13, payload=tv_payload()[:-8]), "its header describes"),
    ("count above 16", lambda: promote256(state_bytes(), 13, payload=tv_payload(count=17)), "1 to 16"),
    ("count 0", lambda: promote256(state_bytes(), 13, payload=tv_payload(count=0)), "1 to 16"),
    ("duplicate tag", lambda: promote256(state_bytes(), 13, payload=tv_payload(((1, 2.0), (1, 3.0)))), "twice"),
    ("negative viscosity", lambda: promote256(state_bytes(), 13, payload=tv_payload(((1, -1.0),))), "negative"),
    ("NaN viscosity", lambda: promote256(state_bytes(), 13, payload=tv_payload(((1, float("nan")),))), "not finite"),
    ("reserved", lambda: promote256(state_bytes(), 13, payload=tv_payload(reserved=1)), "reserved"),
    ("unused entry not zero", lambda: promote256(state_bytes(), 13, payload=tv_payload(tail=((2, 2.0),))), "unused"),
    ("section 17 refused", lambda: promote256(state_bytes(), 13, s17=viscosity_payload(nu=-1.0)), "section 17"),
    ("section 17 missing", lambda: promote256(state_bytes(), 13)[:-(16 + 136 + 4) - (16 + 16 + 4)] + section(20, tv_payload()), "bytes"),
    ("sections 18 and 19 together", lambda: promote256(state_bytes(), 13, with18=True, with19=True), "surface tension"),
    ("section 19 with bodies", lambda: promote256(v8_bytes(BODIES), 15, with19=True), "floating bodies"),
] + [(f"version {v}", (lambda v=v: promote256(state_bytes(), 13, version=v)), "version") for v in (129, 200, 255, 257, 512)])
def test_malformed_version_256_files_are_parse_errors(tmp_path, case, make, needle):
    rc, msg = parse_error(tmp_path, make())
    assert rc == BLUB_ERR_PARSE, (case, rc, msg)
    assert needle in msg, (case, msg)
