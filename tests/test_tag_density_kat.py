"""Liquids of different densities on the host (DESIGN.md §8 "Liquids of different densities"): the restatement of tests/tag_density_ref.py
against independent evaluations and pcg_ref, the hydrostatic balance the weighted solve exists for, the scene key and the version-128
state file."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import pcg_ref
from tests import tag_density_ref as T
from tests import util
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_mesh_bodies_kat import v16_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes, write
from tests.test_surface_tension_kat import promote64, st_payload

BLUB_ERR_PARSE = 5
f32 = np.float32


def random_marker(rng, shape, fluid=0.5, solid=0.1):
    m = np.where(rng.random(shape) < fluid, T.FLUID, np.where(rng.random(shape) < solid / (1 - fluid), T.SOLID, T.AIR)).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = (T.SOLID,) * 6
    return m


# ---- cell density ---------------------------------------------------------------------------------------------------------------
def test_cell_density_against_an_independent_evaluation_and_a_shuffle():
    rng = np.random.default_rng(5)
    shape = (8, 10, 12)
    n = 4000
    pos = np.zeros((n, 4), f32)
    pos[:, 0] = rng.uniform(0.2, 11.9, n)
    pos[:, 1] = rng.uniform(0.2, 9.9, n)
    pos[:, 2] = rng.uniform(0.2, 7.9, n)
    tags = rng.choice(np.array([0, 1, 2, 3, 99], dtype=np.uint32), n)
    table = {1: 0.8, 2: 2.5, 3: 0.125}
    marker = np.full(shape, T.AIR, np.int8)
    marker.ravel()[T.particle_cells(pos, shape)] = T.FLUID
    marker[0], marker[-1], marker[:, 0], marker[:, -1], marker[:, :, 0], marker[:, :, -1] = (T.SOLID,) * 6
    got = T.cell_density(pos, tags, table, marker)
    # independent: per cell, a Python loop over its particles with exact integers
    sums, counts = {}, {}
    for k in range(n):
        x, y, z = (min(int(min(max(float(pos[k, a]), 1.0), d - 1)), d - 1) for a, d in ((0, 12), (1, 10), (2, 8)))
        c = (z, y, x)
        rho = table.get(int(tags[k]), 1.0)
        sums[c] = sums.get(c, 0) + int(round(float(f32(rho)) * 2 ** 20))
        counts[c] = counts.get(c, 0) + 1
    mixed = 0
    for c in zip(*np.nonzero(marker == T.FLUID)):
        want = f32(sums[c] / (counts[c] * 2.0 ** 20))
        assert got[c].view(np.uint32) == want.view(np.uint32)
        mixed += want not in (f32(1), f32(0.8), f32(2.5), f32(0.125))
    assert mixed > 50
    assert not got[marker != T.FLUID].any()
    perm = rng.permutation(n)
    assert np.array_equal(T.cell_density(pos[perm], tags[perm], table, marker).view(np.uint32), got.view(np.uint32))


def test_the_fixed_point_of_a_density_is_its_exact_scaled_value_rounded_once():
    from fractions import Fraction
    for rho in (0.125, 0.8, 1.0, 2.0, 7.99, 8.0):
        exact = Fraction(float(f32(rho))) * 2 ** 20  # the float32 product is exact: a power-of-two scale
        assert Fraction(float(f32(rho) * f32(2 ** 20))) == exact
        assert T.q_of(rho) == round(exact) <= 2 ** 23


# ---- operator -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_with_every_density_one_the_operator_is_the_constant_density_one(seed):
    rng = np.random.default_rng(seed)
    m = random_marker(rng, (10, 12, 16))
    rho = np.where(m == T.FLUID, f32(1), f32(0)).astype(f32)
    beta, D, inv = T.coefficients(m, rho)
    diag, fl = pcg_ref.system(m)
    assert np.array_equal(D, np.where(fl, diag, 0).astype(f32))
    assert np.array_equal(inv.view(np.uint32), np.where(fl, pcg_ref.C_INV_DIAG2[np.minimum(diag, 7)], f32(1)).view(np.uint32))
    x = np.where(fl, rng.standard_normal(m.shape), 0.0)
    assert np.array_equal(T.apply_w(beta, D, fl, x), pcg_ref.apply_A(diag, fl, x)[0])
    x32 = x.astype(f32)
    # pcg_ref.emulate32's A, restated on the same x
    pz = np.pad(x32, 1)
    s6 = ((pz[1:-1, 1:-1, :-2] + pz[1:-1, 1:-1, 2:]) + (pz[1:-1, :-2, 1:-1] + pz[1:-1, 2:, 1:-1])) + (pz[:-2, 1:-1, 1:-1] + pz[2:, 1:-1, 1:-1])
    want = np.where(fl, diag.astype(f32) * x32 - s6, f32(0)).astype(f32)
    assert np.array_equal(T.apply_w32(beta, D, fl, x32).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("seed", [4, 5, 6])
def test_the_weighted_matrix_is_symmetric_positive_definite(seed):
    rng = np.random.default_rng(seed)
    m = random_marker(rng, (9, 11, 13), fluid=0.6, solid=0.0)  # every FLUID component then touches AIR: no null space
    rho = np.where(m == T.FLUID, rng.choice(np.array([0.5, 0.8, 1.0, 1.5, 2.0], dtype=f32), m.shape), f32(0)).astype(f32)
    beta, D, inv = T.coefficients(m, rho)
    fl = m == T.FLUID
    A, idx = T.matrix(beta, D, fl)
    assert abs(A - A.T).max() == 0
    x = np.where(fl, rng.standard_normal(m.shape), 0.0)
    assert np.allclose((A @ x.ravel()[idx]), T.apply_w(beta, D, fl, x).ravel()[idx], rtol=1e-12, atol=1e-12)
    assert np.linalg.eigvalsh(A.toarray()).min() > 0


# ---- hydrostatic balance --------------------------------------------------------------------------------------------------------
def hydrostatic(ratio, weighted=True, shape=(6, 24, 8), split=10, top=18, g_dt=-8.0):
    m = np.full(shape, T.AIR, np.int8)
    m[:, 1:top, :] = T.FLUID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = (T.SOLID,) * 6
    rho = np.where(m == T.FLUID, f32(1.0), f32(0)).astype(f32)
    rho[:, 1:split, :] = np.where(m[:, 1:split, :] == T.FLUID, f32(ratio), f32(0))
    if not weighted:
        rho = np.where(m == T.FLUID, f32(1), f32(0)).astype(f32)
    beta, D, _ = T.coefficients(m, rho, np.float64)
    fl = m == T.FLUID
    u = [np.zeros(shape), np.zeros(shape), np.zeros(shape)]
    for c in range(3):  # u* as the P2G finish leaves it: gravity on the y faces with a FLUID side
        if c == 1:
            u[c] = np.where(fl | (T._shift(m, 1, +1, T.SOLID) == T.FLUID), g_dt, 0.0)
    b = T.divergence(u, m)
    A, idx = T.matrix(beta, D, fl)
    p = np.zeros(shape)
    p.ravel()[idx] = T.solve64(A, b.ravel()[idx])
    return m, rho, beta, u, p


@pytest.mark.parametrize("ratio", [2.0, 0.8, 0.5])
def test_the_weighted_solve_holds_layers_at_rest(ratio):
    m, rho, beta, u, p = hydrostatic(ratio)
    unew = T.project64(u, m, beta, p)
    for c in range(3):  # relative to the largest face velocity u* holds
        assert np.abs(unew[c]).max() <= 1e-12 * 8.0, (c, np.abs(unew[c]).max())
    d = p[2:-2, :-1, 2:-2] - p[2:-2, 1:, 2:-2]
    lower, upper = d[:, 3:8, :].mean(), d[:, 11:16, :].mean()
    assert abs(upper / lower - 1.0 / float(f32(ratio))) < 1e-9  # the density ratio of the float32 densities
    # with one density the pressure holds the column too, but its gradient does not change at the interface: it is not the pressure of
    # two liquids, and the weighted projection of it leaves the heavier layer moving
    m1, _, beta1, u1, p1 = hydrostatic(ratio, weighted=False)
    d1 = p1[2:-2, :-1, 2:-2] - p1[2:-2, 1:, 2:-2]
    assert abs(d1[:, 11:16, :].mean() / d1[:, 3:8, :].mean() - 1.0) < 1e-9
    wrong = T.project64(u, m, beta, p1)
    assert np.abs(wrong[1]).max() > 0.1


# ---- scene key ------------------------------------------------------------------------------------------------------------------
def scene_with(tmp_path, value, extra=None):
    sc = json.load(open(util.scene_path("dam_small")))
    if value is not None:
        sc["fluid"]["tag_densities"] = value
    sc["fluid"].update(extra or {})
    p = tmp_path / "densities.json"
    p.write_text(json.dumps(sc))
    return str(p)


def test_the_scene_key_is_read():
    assert F.scene_tag_densities(util.scene_path("dam_small")) == {}
    assert F.scene_tag_densities(util.scene_path("oil_water_small")) == {1: float(f32(0.8))}


@pytest.mark.parametrize("value", [
    "oil", {"tag": 1}, [1.0], [{"tag": 1}], [{"relative_density": 0.8}], [{"tag": -1, "relative_density": 0.8}],
    [{"tag": 1.5, "relative_density": 0.8}], [{"tag": 1, "relative_density": "light"}], [{"tag": 1, "relative_density": 0.1}],
    [{"tag": 1, "relative_density": 9.0}], [{"tag": 1, "relative_density": 0.49}], [{"tag": 1, "relative_density": 2.01}],
    [{"tag": 1, "relative_density": 1e39}],
    [{"tag": 1, "relative_density": 0.8}, {"tag": 1, "relative_density": 0.9}],
    [{"tag": k, "relative_density": 1.0} for k in range(17)],
])
def test_the_scene_key_refuses_bad_values(tmp_path, value):
    p = scene_with(tmp_path, value)
    L = F.lib()
    assert L.blub_scene_info(os.fsencode(p), F.SceneInfo()) == BLUB_ERR_PARSE
    assert L.blub_scene_tag_densities(os.fsencode(p), None, 0, F.C.byref(F.C.c_uint32())) == BLUB_ERR_PARSE


def test_the_scene_key_refuses_floating_bodies(tmp_path):
    body = {"shape": "box", "position": {"x": 0.16, "y": 0.2, "z": 0.16}, "half_extent": {"x": 0.02, "y": 0.02, "z": 0.02}, "relative_density": 0.9}
    p = scene_with(tmp_path, [{"tag": 1, "relative_density": 0.8}], {"bodies": [body]})
    assert F.lib().blub_scene_info(os.fsencode(p), F.SceneInfo()) == BLUB_ERR_PARSE
    assert F.scene_tag_densities(scene_with(tmp_path, [{"tag": 1, "relative_density": 0.8}], {"bodies": []})) == {1: float(f32(0.8))}


def test_the_scene_key_refuses_surface_tension(tmp_path):
    p = scene_with(tmp_path, [{"tag": 1, "relative_density": 0.8}], {"surface_tension": 1e-5})
    assert F.lib().blub_scene_info(os.fsencode(p), F.SceneInfo()) == BLUB_ERR_PARSE
    assert F.scene_tag_densities(scene_with(tmp_path, [{"tag": 1, "relative_density": 0.8}], {"surface_tension": 0.0})) == {1: float(f32(0.8))}


# ---- state file version 128 -----------------------------------------------------------------------------------------------------
def td_payload(entries=((1, 0.8),), count=None, reserved=0, tail=()):
    out = struct.pack("<II", len(entries) if count is None else count, reserved)
    rows = list(entries) + list(tail)
    for tag, rho in rows:
        out += struct.pack("<If", tag, rho)
    return out + bytes(8 * (16 - len(rows)))


def promote128(base, num_sections, viscous=False, payload=None, tail=b"", with18=False):
    data = promote64(base, num_sections, viscous=viscous, version=128, payload=td_payload() if payload is None else payload, tail=tail)
    # promote64 wrote the setting as section 18: rename it 19 (its checksum covers the payload only)
    head_at = len(data) - len(tail) - (16 + len(td_payload() if payload is None else payload) + 4)
    data = bytearray(data)
    data[head_at:head_at + 4] = struct.pack("<I", 19)
    if with18:  # a surface tension section in front of it
        from tests.test_state_file import section
        data = data[:head_at] + section(18, st_payload()) + data[head_at:]
    return bytes(data)


BASES = {"13 sections": (lambda: state_bytes(), 13), "flow section": (lambda: state_bytes() + section(14, bytes(1056)), 14)}


def with_precond_mode(data, mode):
    """The file with the header's precond_mode (offset 112) set and the header checksum renewed."""
    data = bytearray(data)
    data[112:116] = struct.pack("<i", mode)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    return bytes(data)


@pytest.mark.parametrize("viscous", [False, True])
@pytest.mark.parametrize("base", sorted(BASES))
def test_version_128_written_from_the_documented_layout_is_accepted(tmp_path, base, viscous):
    make, nb = BASES[base]
    info = F.state_info(write(tmp_path, promote128(make(), nb + 1 + viscous, viscous)))
    assert info.format_version == 128


@pytest.mark.parametrize("case, make, needle", [
    ("truncated section 19", lambda: promote128(state_bytes(), 14, payload=td_payload()[:-8]), "its header describes"),
    ("count above 16", lambda: promote128(state_bytes(), 14, payload=td_payload(count=17)), "1 to 16"),
    ("count 0", lambda: promote128(state_bytes(), 14, payload=td_payload(count=0)), "1 to 16"),
    ("duplicate tag", lambda: promote128(state_bytes(), 14, payload=td_payload(((1, 0.8), (1, 2.0)))), "twice"),
    ("density out of range", lambda: promote128(state_bytes(), 14, payload=td_payload(((1, 9.0),))), "outside"),
    ("density NaN", lambda: promote128(state_bytes(), 14, payload=td_payload(((1, float("nan")),))), "outside"),
    ("reserved", lambda: promote128(state_bytes(), 14, payload=td_payload(reserved=1)), "reserved"),
    ("unused entry not zero", lambda: promote128(state_bytes(), 14, payload=td_payload(count=1, entries=((1, 0.8),), tail=((2, 2.0),))), "unused"),
    ("section 18 with section 19", lambda: promote128(state_bytes(), 15, with18=True), "its header describes"),
    ("precond_mode 1", lambda: with_precond_mode(promote128(state_bytes(), 14), 1), "precond_mode 0"),
    ("floating bodies", lambda: promote128(v8_bytes(BODIES), 16), "floating bodies"),
    ("mesh bodies", lambda: promote128(v16_bytes(), 17), "floating bodies"),
] + [(f"version {v}", (lambda v=v: bytes(bytearray(promote128(state_bytes(), 14)[:8]) + struct.pack("<I", v) + promote128(state_bytes(), 14)[12:])),
      "version") for v in (65, 100, 127, 256)])
def test_malformed_version_128_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    assert rc == BLUB_ERR_PARSE, (case, rc)
    assert needle in L.blub_last_error().decode(), (case, L.blub_last_error().decode())
