"""CPU: tests/step_ref.py pinned before any GPU is involved -- it reproduces the known answers of test_stage_kat.py and test_transfer_kat.py,
the oracle stays within its bounds on rough inputs (salt-and-pepper markers, independent random faces, particles on every plane the kernels
decide at), and its bounds catch errors a tolerance comparison with the oracle lets through.

The rough inputs and the stage driver here are shared with tests/test_gpu_step_ref.py, which runs the same checks on the CUDA kernels."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import step_ref as R
from tests import test_stage_kat as SK
from tests import test_transfer_kat as TK
from tests.util import DT

f32 = np.float32
FILLS = [0.03, 0.5, 0.97]
KAT_SHAPES = [(8, 48, 48), (48, 8, 48), (264, 8, 8)]  # three rows of test_gpu_shapes.SHAPES


# ------------------------------------------------------------------------------------------------ rough inputs
def rough_inputs(dims, fill, seed, with_vox=True):
    """Salt-and-pepper marker (FLUID with probability `fill`, SOLID 10 % of the rest, borders SOLID), every face an independent uniform value
    in [-40, 40] cells/s, random pressures and residuals, displacement fields of up to 0.6 cells (stage 13), and an fp16 solid volume whose w > 0 on half of the interior
    SOLID cells (random velocities; a third of them with |s.x|, |s.y|, |s.z| tied pairwise or all three)."""
    nx, ny, nz = dims
    rng = np.random.default_rng(seed)
    shape = (nz, ny, nx)
    m = np.full(shape, R.AIR, dtype=np.int8)
    r = rng.random(shape)
    m[r < fill] = R.FLUID
    m[(r >= fill) & (rng.random(shape) < 0.1)] = R.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = R.SOLID, R.SOLID, R.SOLID, R.SOLID, R.SOLID, R.SOLID
    inp = {"dims": dims, "marker": m, "u": [rng.uniform(-40, 40, shape).astype(f32) for _ in range(3)],
           "p": rng.uniform(-20, 20, shape).astype(f32), "rhs": rng.uniform(-5, 5, shape).astype(f32), "vox": None,
           "disp": [rng.uniform(-0.6, 0.6, shape).astype(f32) for _ in range(3)]}
    if with_vox:
        vox = np.zeros(shape + (4,), dtype=np.float16)
        interior = np.zeros(shape, dtype=bool)
        interior[1:-1, 1:-1, 1:-1] = True
        sel = (m == R.SOLID) & interior & (rng.random(shape) < 0.5)
        k = int(sel.sum())
        v = rng.uniform(-20, 20, (k, 3))
        tie = rng.integers(0, 6, k)  # 0: x = y, 1: y = z, 2: x = z, 3: all three, else none
        s = np.sign(rng.uniform(-1, 1, (k, 3)))
        for t, (a, b) in enumerate(((0, 1), (1, 2), (0, 2))):
            v[tie == t, b] = s[tie == t, b] * np.abs(v[tie == t, a])
        v[tie == 3, 1] = s[tie == 3, 1] * np.abs(v[tie == 3, 0])
        v[tie == 3, 2] = s[tie == 3, 2] * np.abs(v[tie == 3, 0])
        vox[sel, :3] = v.astype(np.float16)
        vox[sel, 3] = rng.choice([0.5, 1.0, 2.0], k).astype(np.float16)
        inp["vox"] = vox
    return inp


def rough_particles(inp, seed, per_cell=2, outside=True):
    """Particles: random ones in FLUID cells; ones exactly on cell planes (k), dual-cell planes (k + 0.5), both clamp planes and one ulp either
    side of them; random ones inside SOLID cells with w > 0 (eaten); four outside the domain (outside = True: the kernels clamp their
    corner indices to the grid, where the oracle reads 0 past it as the shader's texelFetch does).  Random APIC rows."""
    nx, ny, nz = dims = inp["dims"]
    S = np.array(dims)
    rng = np.random.default_rng(seed)
    m = inp["marker"]
    fl = np.argwhere(m == R.FLUID)[:, ::-1]
    parts = [np.repeat(fl, per_cell, axis=0) + rng.random((len(fl) * per_cell, 3))]
    lo_pl, hi_pl = f32(1.001), S.astype(f32) - f32(1.001)
    for ax in range(3):
        vals = [f32(1.0), f32(2.0), f32(S[ax] - 2), f32(1.5), f32(2.5), f32(S[ax] // 2 + 0.5), lo_pl, hi_pl[ax]]
        vals += [np.nextafter(lo_pl, f32(0)), np.nextafter(lo_pl, f32(9)), np.nextafter(hi_pl[ax], f32(0)), np.nextafter(hi_pl[ax], f32(1e9))]
        for v in vals:
            q = 1.0 + rng.random((8, 3)) * (S - 2)
            q[:, ax] = v
            parts.append(q)
    if inp["vox"] is not None:
        eat = np.argwhere(inp["vox"][..., 3] > 0)[:, ::-1]
        if len(eat):
            parts.append(eat + rng.random(eat.shape))
    if outside:
        parts.append(np.array([[-5.0, 3.0, 3.0], [S[0] + 8.0, 3.0, 3.0], [3.0, -1e6, 3.0], [3.0, 3.0, 1e6]]))
    p = np.concatenate(parts).astype(f32)
    pos = np.c_[p, rng.uniform(-1, 1, len(p))].astype(f32)
    rows = [rng.normal(0, 10.0, (len(p), 4)).astype(f32) for _ in range(3)]
    return pos, rows


# ------------------------------------------------------------------------------------------------ stage driver (oracle here, CUDA in the GPU file)
class OracleStages:
    KEEPS_W = False

    def __init__(self, dims, capacity):
        self.f = O.OracleFluid(*dims, capacity)
        self.f.set_gravity_grid([0.0, 0.0, 0.0])
        self.f.set_rebin_frequency(0)

    def put(self, inp, which, pos=None, rows=None, marker=None):
        f = self.f
        f.set_voxels(R.voxel_values(inp["vox"], inp["marker"].shape) if inp["vox"] is not None else np.zeros(inp["marker"].shape + (4,), np.float32))
        f.grid(O.ARR_MARKER)[:] = inp["marker"] if marker is None else marker
        for c, a in enumerate((O.ARR_UX, O.ARR_UY, O.ARR_UZ)):
            f.grid(a)[:] = inp["u"][c]
        f.grid(O.ARR_P_VEL if which == 0 else O.ARR_P_DEN)[:] = inp["p"]
        f.grid(O.ARR_RESIDUAL)[:] = inp["rhs"]
        if pos is not None:
            f.set_particles(pos, *(rows or (None, None, None)))

    def run(self, a, b):
        self.f.step_stages(DT, a, b)

    def u(self):
        return [self.f.grid(a).copy() for a in (O.ARR_UX, O.ARR_UY, O.ARR_UZ)]

    def residual(self):
        return self.f.grid(O.ARR_RESIDUAL).copy()

    def marker(self):
        return self.f.grid(O.ARR_MARKER).copy()

    def particles(self):
        return self.f.particles().copy(), [self.f.particles(a).copy() for a in (O.ARR_ROWX, O.ARR_ROWY, O.ARR_ROWZ)]


def check_stages(backend, inp, pos, rows, stages, unwritten=True, report=None):
    """Run each stage of `stages` on its own from the inputs and compare every element with tests/step_ref.py.  unwritten = False: the
    elements stages 4 and 11 do not write are not compared (the oracle's passes visit every cell).  Fills report[stage] with the err / bound
    ratios, the branch counts and the margin particles that took another branch."""
    report = {} if report is None else report
    m = inp["marker"]
    for st in stages:
        rec = report.setdefault(st, {"ratios": [], "counts": {}, "alt_taken": 0})
        if st == 1:
            backend.put(inp, 0)
            backend.run(1, 2)
            rec["ratios"].append(R.check_grid(backend.residual(), R.divergence(m, inp["u"], inp["vox"], inp["rhs"]), f"stage 1 {inp['dims']}"))
        elif st in (4, 11):
            backend.put(inp, 0 if st == 4 else 1)
            backend.run(st, st + 1)
            ref = R.project(m, inp["u"], inp["p"], inp["vox"]) if st == 4 else R.position_change(m, inp["u"], inp["p"], DT)
            for c, got in enumerate(backend.u()):
                rec["ratios"].append(R.check_grid(got, ref[c], f"stage {st} u[{c}] {inp['dims']}", unwritten=unwritten))
        elif st in (5, 12):
            backend.put(inp, 0)
            backend.run(st, st + 1)
            ref = R.extrapolate(m, inp["u"])
            for c, got in enumerate(backend.u()):
                rec["ratios"].append(R.check_grid(got, ref[c], f"stage {st} u[{c}] {inp['dims']}"))
        elif st == 7:
            backend.put(inp, 0, pos, rows)
            backend.run(6, 8)
            ref = R.advect(inp["u"], inp["vox"], pos, DT)
            gp, gr = backend.particles()
            r, alt = R.check_particles(gp, ref, f"stage 7 {inp['dims']}", got_rows=gr, got_marker=backend.marker(), keeps_w=backend.KEEPS_W)
            rec["ratios"].append(r)
            rec["alt_taken"] += alt
            for k, v in ref["counts"].items():
                rec["counts"][k] = rec["counts"].get(k, 0) + v
        elif st == 13:
            backend.put(dict(inp, u=inp["disp"]), 1, pos, rows)
            backend.run(13, 14)
            ref = R.correct(inp["disp"], m, pos)
            gp, _ = backend.particles()
            r, alt = R.check_particles(gp, ref, f"stage 13 {inp['dims']}", keeps_w=backend.KEEPS_W)
            rec["ratios"].append(r)
            rec["alt_taken"] += alt
            for k, v in ref["counts"].items():
                rec["counts"][k] = rec["counts"].get(k, 0) + v
    return report


def print_report(what, report):
    for st, rec in sorted(report.items()):
        r = np.concatenate([np.ravel(a) for a in rec["ratios"]]) if rec["ratios"] else np.zeros(1)
        r = r[r > 0] if (r > 0).any() else np.zeros(1)
        print(f"{what} stage {st}: error / bound median {np.median(r):.3f} max {r.max():.3f}; counts {rec['counts']}; "
              f"margin particles on another branch: {rec['alt_taken']}")


# ------------------------------------------------------------------------------------------------ 1. known answers
def test_reference_reproduces_the_grid_stage_known_answers():
    """test_stage_kat.py's closed forms, from the reference: trace, projection by +K, position change K dt, a constant extrapolated."""
    m = SK.block_marker()
    rhs = R.divergence(m, [SK.face_field(c) for c in range(3)], None, np.zeros(m.shape, f32))
    assert np.abs(rhs["want"][m == R.FLUID] - np.trace(SK.A)).max() <= 2e-4
    proj = R.project(m, [np.full(m.shape, SK.B[c], f32) for c in range(3)], SK.cell_pressure(), None)
    pc = R.position_change(SK.block_marker(lo=1, hi=24), [np.zeros(m.shape, f32)] * 3, SK.cell_pressure(), DT)
    for c in range(3):
        ff = SK.fluid_fluid_faces(m, c)
        assert np.abs(proj[c]["want"][ff] - (SK.B[c] + SK.K[c])).max() <= 1e-4
        ff1 = SK.fluid_fluid_faces(SK.block_marker(lo=1, hi=24), c)
        assert np.abs(pc[c]["want"][ff1] - f32(SK.K[c]) * f32(DT)).max() <= 2e-6
    ms, vox = SK.shell_marker_and_vox()
    proj = R.project(ms, [np.full(ms.shape, SK.B[c], f32) for c in range(3)], SK.cell_pressure(), vox)
    pcs = R.position_change(ms, [np.zeros(ms.shape, f32)] * 3, SK.cell_pressure(), DT)
    for c in range(3):
        want, lo, hi = SK.face_value_next_to_solid(ms, vox, c)
        assert np.array_equal(proj[c]["bits"][lo | hi], want[lo | hi])
        assert (pcs[c]["bits"][lo | hi] == 0).all()
    # the divergence next to the moving shell: the solid terms replace the faces on the solid side
    u = [SK.face_field(c) for c in range(3)]
    d = R.divergence(ms, u, vox, np.zeros(ms.shape, f32))
    want = np.zeros(ms.shape)
    for c in range(3):
        ax = 2 - c
        v = vox[..., c].astype(np.float64)
        plus = np.where(np.roll(ms, -1, axis=ax) == O.SOLID, np.roll(v, -1, axis=ax), u[c])
        minus = np.where(np.roll(ms, 1, axis=ax) == O.SOLID, np.roll(v, 1, axis=ax), np.roll(u[c], 1, axis=ax))
        want += plus - minus
    fl = ms == R.FLUID
    assert np.abs(d["want"][fl] - want[fl]).max() <= 2e-4
    # a constant on the valid faces is copied into the first ring, garbage elsewhere is kept
    fl = m == R.FLUID
    rng = np.random.default_rng(0)
    uu = []
    for c in range(3):
        f = rng.uniform(50, 60, m.shape).astype(f32)
        f[R.valid_faces(m, c)] = f32(SK.B[c])
        uu.append(f)
    ex = R.extrapolate(m, uu)
    for c in range(3):
        w = ex[c]["written"]
        assert w.sum() > 1000 and np.abs(ex[c]["want"][w] - SK.B[c]).max() <= 4 * R.U * abs(SK.B[c]) * 8
        assert np.array_equal(ex[c]["bits"][~w], uu[c][~w])


def test_reference_reproduces_the_transfer_known_answers():
    """test_transfer_kat.py's G2P closed forms: a linear field gives v(x0) and the columns of A as the rows; a constant field moves every
    particle by dt b and leaves zero Jacobian rows."""
    pos, _ = TK.g2p_setup()
    u = [TK.linear_field(TK.A_ANY, TK.face_centres(c))[..., c].astype(f32) for c in range(3)]
    ref = R.advect(u, None, pos, 1e-3)
    rows = [ref["nat"]["rows"][c].v for c in range(3)]
    TK.check_g2p_linear(pos, rows)
    pos, _ = TK.g2p_setup(seed=4)
    ref = R.advect([np.full((TK.N,) * 3, f32(TK.B_VEC[c])) for c in range(3)], None, pos, DT)
    want = pos[:, :3].astype(np.float64) + DT * TK.B_VEC
    assert np.abs(ref["nat"]["pos"].v - want).max() <= 4e-6 * 24
    for c in range(3):
        r = ref["nat"]["rows"][c].v
        assert np.abs(r[:, :3]).max() == 0.0 and np.abs(r[:, 3] - TK.B_VEC[c]).max() <= 1e-6 * 6


# ------------------------------------------------------------------------------------------------ 2. the oracle within the bounds
@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("dims", KAT_SHAPES, ids=[f"{a}x{b}x{c}" for a, b, c in KAT_SHAPES])
def test_oracle_within_the_reference_bounds(dims, fill):
    """Every stage of the oracle, run on its own from rough inputs, within the reference's per-element bounds; the oracle's grid passes visit
    every cell, so the elements the kernels do not write are compared only where the reference writes them."""
    inp = rough_inputs(dims, fill, seed=int(fill * 100) + dims[0])
    pos, rows = rough_particles(inp, seed=3, outside=False)
    b = OracleStages(dims, len(pos))
    rep = check_stages(b, inp, pos, rows, [1, 4, 5, 7, 11, 12, 13], unwritten=False)
    print_report(f"oracle {dims} fill {fill}", rep)
    c7 = rep[7]["counts"]
    assert c7["eaten_x"] + c7["eaten_y"] + c7["eaten_z"] > 0 and c7["wall"] > 0 and rep[13]["counts"]["hit"] > 0, (c7, rep[13]["counts"])


def test_oracle_extrapolation_and_divergence_write_only_what_the_reference_writes():
    """The oracle's extrapolation and divergence leave every element outside their written set bit for bit (the stage 4 / 11 passes are
    compared written-set only above)."""
    inp = rough_inputs((48, 8, 48), 0.5, seed=5)
    b = OracleStages((48, 8, 48), 8)
    check_stages(b, inp, None, None, [1, 5, 12], unwritten=True)


# ------------------------------------------------------------------------------------------------ 3. the bounds catch errors
def _oracle_case(dims=(48, 8, 48), fill=0.5, seed=21):
    inp = rough_inputs(dims, fill, seed)
    pos, rows = rough_particles(inp, seed=4, outside=False)
    return inp, pos, rows


def test_a_face_replaced_by_its_neighbour_is_caught():
    """The oracle's extrapolation with one written face replaced by its in-plane neighbour's value: check_grid names that face."""
    inp, _, _ = _oracle_case()
    b = OracleStages(inp["dims"], 8)
    b.put(inp, 0)
    b.run(5, 6)
    u = b.u()
    ref = R.extrapolate(inp["marker"], inp["u"])
    R.check_grid(u[1], ref[1], "unchanged")
    w = np.argwhere(ref[1]["written"])
    for z, y, x in w:
        if x + 1 < u[1].shape[2] and abs(u[1][z, y, x + 1] - u[1][z, y, x]) > 1.0:
            break
    bad = u[1].copy()
    bad[z, y, x] = bad[z, y, x + 1]
    with pytest.raises(AssertionError, match=rf"\[z, y, x\] = \({z}, {y}, {x}\)"):
        R.check_grid(bad, ref[1], "mutant")
    # the averages of only the four edge neighbours
    edges = R.extrapolate(inp["marker"], inp["u"], mutant="edges")
    with pytest.raises(AssertionError, match="rounded elements beyond their bound"):
        R.check_grid(np.where(edges[1]["written"], edges[1]["want"], edges[1]["bits"]).astype(f32), ref[1], "edges")


@pytest.mark.parametrize("mutant", ["cy_iy", "b17_fixed"])
def test_a_swapped_fraction_and_a_fixed_b17_are_caught(mutant):
    """The oracle's advection passes; an APIC row built with iy in place of iz, or an RK4 that advances component k's interpolants by
    step[axis] (B17 "fixed"), fails check_particles with the particle and the element named."""
    inp, pos, rows = _oracle_case()
    b = OracleStages(inp["dims"], len(pos))
    rep = check_stages(b, inp, pos, rows, [7])
    assert rep[7]["counts"]["hit"] > 0
    ref = R.advect(inp["u"], inp["vox"], pos, DT)
    mut = R.advect(inp["u"], inp["vox"], pos, DT, mutant=mutant)
    gp = np.c_[mut["nat"]["pos"].v, pos[:, 3]].astype(f32)
    gr = [mut["nat"]["rows"][k].v.astype(f32) for k in range(3)]
    what = "row" if mutant == "cy_iy" else "(pos|row)"
    with pytest.raises(AssertionError, match=rf"particle \d+, {what}\d?\[\d\]"):
        R.check_particles(gp, ref, "mutant", got_rows=gr)
