"""CPU: known answers of the solid load probes (DESIGN.md §8, "Solid load probes"): the NumPy restatement on hand-built fields, the
fixed-point quantisation against exact rational rounding and the documented exactness range, the [0, dim] box clamp against add_cube's, and
the scene key "load_probes" as blub_scene_info parses it.  No GPU needed."""
import json
import os
from fractions import Fraction

import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import flow_ref, load_ref, util

BLUB_ERR_INVALID_ARGUMENT, BLUB_ERR_PARSE = 1, 5
AIR = -1


# The velocity solve's volume holds -p dt / density (divergence_remove subtracts p_cell - p_next from a face): the fields below store the
# negated pressure, q = -p_vel * inv_dt.
def grid(n=8, fill=AIR):
    return np.full((n, n, n), fill, dtype=np.int8), np.zeros((n, n, n), dtype=np.float32)


# ---- the restatement on hand-built fields --------------------------------------------------------------------------------
def test_one_solid_cell_with_six_fluid_neighbours():
    m, p = grid()
    m[4, 4, 4] = load_ref.SOLID
    pressures = {(-1, 0): 1.0, (1, 0): 2.0, (-1, 1): 3.0, (1, 1): 4.0, (-1, 2): 5.0, (1, 2): 6.0}  # (direction, axis x/y/z): p * dt / rho
    for (d, a), v in pressures.items():
        c = [4, 4, 4]
        c[a] += d
        m[c[2], c[1], c[0]] = load_ref.FLUID
        p[c[2], c[1], c[0]] = -v
    # inv_dt 2: q = 2 p.  The -x neighbour pushes towards +x, the +x one towards -x: F_a = q(-) - q(+) = -2 on every axis
    rec = load_ref.solid_loads(m, p, 2.0, (4, 4, 4), (5, 5, 5), (4.5, 4.5, 4.5))
    assert rec == {"wetted_faces": 6, "force_fx": [-2 * 65536] * 3, "torque_fx": [0, 0, 0]}  # every arm is parallel to its force
    # a box around the cell that also holds its neighbours: the fluid cells add nothing, the faces stay 6
    assert load_ref.solid_loads(m, p, 2.0, (3, 3, 3), (6, 6, 6), (4.5, 4.5, 4.5)) == rec
    # a box beside the cell holds no solid: nothing
    assert load_ref.solid_loads(m, p, 2.0, (5, 4, 4), (6, 5, 5), (0, 0, 0)) == {"wetted_faces": 0, "force_fx": [0, 0, 0], "torque_fx": [0, 0, 0]}


def test_a_box_on_border_cells_holds_the_wall():
    """8^3 tank: border cells SOLID, the interior FLUID at q = 3.  The x = 0 wall has 6 x 6 wetted faces; its edge cells touch only walls."""
    m, p = grid(fill=load_ref.SOLID)
    m[1:-1, 1:-1, 1:-1] = load_ref.FLUID
    p[1:-1, 1:-1, 1:-1] = -1.5
    cells = load_ref.probe_cells((8, 8, 8), (-5.0, -1.0, 0.0), (1.0, 100.0, 8.0))
    assert cells == ((0, 0, 0), (1, 8, 8))
    rec = load_ref.solid_loads(m, p, 2.0, *cells, (0.5, 4.0, 4.0))
    # water pushes the x = 0 wall towards -x; the arms (0.5, y - 3.5, z - 3.5) sum to zero in y and z
    assert rec == {"wetted_faces": 36, "force_fx": [-36 * 3 * 65536, 0, 0], "torque_fx": [0, 0, 0]}
    # the whole grid: the six walls cancel
    whole = load_ref.solid_loads(m, p, 2.0, (0, 0, 0), (8, 8, 8), (4.0, 4.0, 4.0))
    assert whole == {"wetted_faces": 6 * 36, "force_fx": [0, 0, 0], "torque_fx": [0, 0, 0]}


def test_a_pivot_off_the_centre():
    """One fluid neighbour above the cell, q = 4: F = (0, -4, 0) at the face centre (4.5, 5, 4.5).  About the origin
    tau = r x F = (-r_z F_y, 0, r_x F_y) = (18, 0, -18)."""
    m, p = grid()
    m[4, 4, 4] = load_ref.SOLID
    m[4, 5, 4] = load_ref.FLUID
    p[4, 5, 4] = -2.0
    rec = load_ref.solid_loads(m, p, 2.0, (4, 4, 4), (5, 5, 5), (0.0, 0.0, 0.0))
    assert rec == {"wetted_faces": 1, "force_fx": [0, -4 * 65536, 0], "torque_fx": [18 * 256, 0, -18 * 256]}
    # about a pivot shifted by (1, 0, 0): tau' = tau - (shift x F) = (18, 0, -18) - (0, 0, -4)
    rec = load_ref.solid_loads(m, p, 2.0, (4, 4, 4), (5, 5, 5), (1.0, 0.0, 0.0))
    assert rec["torque_fx"] == [18 * 256, 0, -14 * 256]


def loop_loads(marker, p_vel, inv_dt, lo, hi, pivot):
    """The rule face by face with float32 scalars: the restatement's vectorised form checked against it."""
    nz, ny, nx = marker.shape
    dims = (nx, ny, nz)
    pivot = [np.float32(v) for v in pivot]
    faces, force, torque = 0, [0, 0, 0], [0, 0, 0]
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                if marker[z, y, x] != load_ref.SOLID:
                    continue
                for a in range(3):
                    for d in (-1, 1):
                        c = [x, y, z]
                        c[a] += d
                        if not 0 <= c[a] < dims[a] or marker[c[2], c[1], c[0]] != load_ref.FLUID:
                            continue
                        q = -(np.float32(p_vel[c[2], c[1], c[0]]) * np.float32(inv_dt))
                        centre = [np.float32(v) + np.float32(0.5) for v in (x, y, z)]
                        centre[a] = np.float32(max(c[a], (x, y, z)[a]))
                        r = [centre[k] - pivot[k] for k in range(3)]
                        f = [np.float32(0)] * 3
                        f[a] = -d * q
                        faces += 1
                        force[a] += round(Fraction(float(f[a])) * 65536)
                        tau = [r[1] * f[2] - r[2] * f[1], r[2] * f[0] - r[0] * f[2], r[0] * f[1] - r[1] * f[0]]  # one product is non-zero
                        torque = [t + round(Fraction(float(np.float32(v))) * 256) for t, v in zip(torque, tau)]
    return {"wetted_faces": faces, "force_fx": force, "torque_fx": torque}


def test_the_restatement_agrees_with_a_face_by_face_loop():
    rng = np.random.default_rng(1)
    m = rng.choice(np.array([load_ref.SOLID, load_ref.FLUID, AIR], dtype=np.int8), (8, 10, 12), p=[0.3, 0.5, 0.2])
    p = (rng.standard_normal(m.shape) * 50).astype(np.float32)
    for lo, hi, pivot in [((0, 0, 0), (12, 10, 8), (6.0, 5.0, 4.0)), ((3, 2, 1), (9, 7, 5), (-3.25, 17.5, 0.1)), ((11, 0, 0), (12, 10, 8), (12, 5, 4))]:
        assert load_ref.solid_loads(m, p, 119.99999, lo, hi, pivot) == loop_loads(m, p, 119.99999, lo, hi, pivot)


# ---- quantisation ---------------------------------------------------------------------------------------------------------
Q_MAX = float(np.nextafter(np.float32(2 ** 22), np.float32(0)))  # the largest |q| below 2^22
R_MAX = float(np.nextafter(np.float32(2 ** 11), np.float32(0)))
EDGES = [0.0, -0.0, 1.0, -1.0, 0.5 / 65536, 1.5 / 65536, 2.5 / 65536, -2.5 / 65536, 2.0 ** -149, 3 * 2.0 ** -18, 1.0001, 1e-3, -123.456,
         Q_MAX, -Q_MAX, 0.5 / 256, 1.5 / 256]


def test_force_quantisation_rounds_the_exact_value_to_nearest_even():
    q = np.asarray(EDGES, dtype=np.float32)
    assert load_ref.force_fixed(q).tolist() == [round(Fraction(float(v)) * 65536) for v in q]
    assert load_ref.force_fixed([0.5 / 65536, 1.5 / 65536, 2.5 / 65536]).tolist() == [0, 2, 2]


def test_torque_quantisation_is_one_float32_product_then_exact_rounding():
    rng = np.random.default_rng(2)
    r = np.concatenate([rng.uniform(-R_MAX, R_MAX, 500), [R_MAX, -R_MAX, 0.5, 1.0 / 3]]).astype(np.float32)
    q = np.concatenate([rng.standard_normal(500) * rng.choice([1e-3, 1.0, 1e3, 1e6], 500), [Q_MAX, Q_MAX, 1.0 / 256, 3.0]]).astype(np.float32)
    want = []
    for a, b in zip(r, q):
        prod = np.float32(np.float64(a) * np.float64(b))  # the float64 product of two float32 is exact: one rounding to float32
        want.append(round(Fraction(float(prod)) * 256))
    assert load_ref.torque_fixed(r, q).tolist() == want
    # the rounding of the product matters: it is not the exact product rounded to 2^-8
    assert load_ref.torque_fixed(np.float32(1.0 / 3), np.float32(3.0)).tolist() == round(Fraction(float(np.float32(np.float32(1.0 / 3) * np.float32(3.0)))) * 256)


def test_sums_stay_exact_in_the_documented_range():
    """|q| < 2^22, |r| < 2^11 and at most 2^21 wetted faces per probe keep every sum below 2^63."""
    faces = 2 ** 21
    f_max = int(load_ref.force_fixed(np.float32(Q_MAX)))
    t_max = int(load_ref.torque_fixed(np.float32(R_MAX), np.float32(Q_MAX)))
    assert f_max == round(Fraction(Q_MAX) * 65536) and faces * f_max < 2 ** 63
    assert faces * t_max < 2 ** 63
    # a torque component collects one product per face, the force component one value: both bounds hold per component
    assert faces * f_max < 2 ** 60 and faces * t_max <= 2 ** 62
    # every per-face value is an integer of at most 41 bits, exact in float64 and in the int64 atomics
    assert max(f_max, t_max) < 2 ** 41


# ---- the box clamp --------------------------------------------------------------------------------------------------------
VALUES = [-1e30, -5.0, -0.0, 0.0, 0.25, 0.999, 1.0, 1.5, 2.0, 7.0, 7.5, 8.0, 8.5, 9.0, 31.0, 31.99, 32.0, 33.0, 1e9, 4294967040.0, 1e30]


@pytest.mark.parametrize("dim", [8, 32, 64])
def test_probe_clamp_is_add_cubes_clamp_widened_to_the_border(dim):
    for v in VALUES:
        c, a = load_ref.clamp_closed(dim, v), flow_ref.clamp_to_grid(dim, v)
        assert 0 <= c <= dim
        if 1 <= c <= dim - 1:
            assert c == a, v
        else:  # only the border values differ: add_cube stops at 1 and dim - 1
            assert (c, a) in ((0, 1), (dim, dim - 1)), v
    # the library's clamp (host only) agrees with the restatement and refuses what set_load_probes refuses
    for mn in VALUES:
        for mx in (0.5, 1.0, 4.0, float(dim), 1e9):
            want = load_ref.probe_cells((dim, dim, dim), (mn, 1.0, 0.0), (mx, dim - 1.0, 1e9))
            if want is None:
                with pytest.raises(F.BlubError):
                    F.load_probe_cells((dim, dim, dim), ((mn, 1.0, 0.0), (mx, dim - 1.0, 1e9)))
            else:
                assert F.load_probe_cells((dim, dim, dim), ((mn, 1.0, 0.0), (mx, dim - 1.0, 1e9))) == want
    for bad in [((float("nan"), 0, 0), (4, 4, 4)), ((0, 0, 0), (4, float("inf"), 4)), ((0, 0, 0), (4, 4, 4), (0, float("nan"), 0)),
                ((3, 3, 3), (3, 5, 5)), ((-4, 0, 0), (0, 4, 4))]:
        with pytest.raises(F.BlubError):
            F.load_probe_cells((dim, dim, dim), bad)


# ---- scene key ------------------------------------------------------------------------------------------------------------
def scene_with(tmp_path, probes, name="s.json"):
    sc = json.load(open(util.scene_path("dam_small")))
    if probes is not ...:
        sc["fluid"]["load_probes"] = probes
    path = str(tmp_path / name)
    with open(path, "w") as f:
        json.dump(sc, f)
    return path, sc


def v3(x, y, z):
    return {"x": x, "y": y, "z": z}


def test_scene_probes_convert_to_grid_cells(tmp_path):
    path, sc = scene_with(tmp_path, [{"min": v3(0.0, 0.0, 0.0), "max": v3(0.01, 0.32, 0.32)},
                                     {"min": v3(0.1, 0.05, 0.1), "max": v3(0.2, 0.15, 0.2), "pivot": v3(0.15, 0.0, -0.01)}])
    scale = np.float32(sc["fluid"]["grid_to_world_scale"])
    got = F.scene_load_probes(path)
    assert len(got) == 2
    for (mn, mx, pv), want in zip(got, sc["fluid"]["load_probes"]):
        wmn = [np.float32(want["min"][a]) / scale for a in "xyz"]
        wmx = [np.float32(want["max"][a]) / scale for a in "xyz"]
        wpv = [np.float32(want["pivot"][a]) / scale for a in "xyz"] if "pivot" in want else [(a + b) * np.float32(0.5) for a, b in zip(wmn, wmx)]
        assert list(mn) == [float(v) for v in wmn] and list(mx) == [float(v) for v in wmx] and list(pv) == [float(v) for v in wpv]
    F.scene_info(path)
    assert F.scene_load_probes(scene_with(tmp_path, ..., "none.json")[0]) == []


BAD = [
    ("not an array", {"min": v3(0, 0, 0), "max": v3(1, 1, 1)}),
    ("entry not an object", [[0, 0, 0]]),
    ("missing max", [{"min": v3(0, 0, 0)}]),
    ("min not a number", [{"min": v3("a", 0, 0), "max": v3(1, 1, 1)}]),
    ("pivot without z", [{"min": v3(0, 0, 0), "max": v3(1, 1, 1), "pivot": {"x": 0, "y": 0}}]),
    ("pivot not an object", [{"min": v3(0, 0, 0), "max": v3(1, 1, 1), "pivot": 3}]),
    ("beyond float", [{"min": v3(0, 0, 0), "max": v3(1e39, 1, 1)}]),
    ("17 probes", [{"min": v3(0, 0, 0), "max": v3(0.1, 0.1, 0.1)}] * 17),
]


@pytest.mark.parametrize("what,probes", BAD, ids=[b[0] for b in BAD])
def test_bad_load_probes_are_parse_errors(tmp_path, what, probes):
    path, _ = scene_with(tmp_path, probes)
    info = F.SceneInfo()
    assert F.lib().blub_scene_info(os.fsencode(path), info) == BLUB_ERR_PARSE, what
    with pytest.raises(F.BlubError):
        F.scene_load_probes(path)
