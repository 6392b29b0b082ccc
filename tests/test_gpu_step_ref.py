"""GPU: every grid pass, the advection and the density correction on their own, element by element against the float64 restatements of
tests/step_ref.py (rough inputs of tests/test_step_ref_kat.py), at particle counts around the particle kernels' grid-stride size, and the
claim of DESIGN section 3.3 (SURVEY B6) that the faces the grid passes leave stale are never read, tested by poisoning them."""
import numpy as np
import pytest

from tests import step_ref as R
from tests.test_gpu_shapes import SHAPE_LIST, fluid_box, sphere_volume
from tests.test_step_ref_kat import FILLS, check_stages, print_report, rough_inputs, rough_particles
from tests.util import DT

STEP_SHAPES = SHAPE_LIST + [(1024, 8, 8)]  # 1024: positions near 1000 cells stretch the u |x| terms
STAGES = [1, 4, 5, 7, 11, 12, 13]


class CudaStages:
    """The stage driver of test_step_ref_kat.py on the CUDA library: inputs through the taps, step_stages(k, k + 1), outputs through the taps."""
    KEEPS_W = True

    def __init__(self, dims, capacity, scatter=True):
        import blub_b200
        from blub_b200 import fluid as F
        self.F = F
        self.f = blub_b200.HybridFluid(*dims, capacity)
        self.f.set_gravity_grid([0.0, 0.0, 0.0])
        self.f.set_rebin_frequency(0)
        self.f.set_transfer_path(scatter)
        self.keep = None

    def put(self, inp, which, pos=None, rows=None, marker=None):
        F, f = self.F, self.f
        if inp["vox"] is not None and self.keep is None:
            import torch
            self.keep = torch.from_numpy(np.ascontiguousarray(inp["vox"], dtype=np.float16)).to("cuda")  # the fluid borrows it
            torch.cuda.synchronize()
            f.set_solid_voxels(self.keep.data_ptr())
        f.upload_grid(F.TAP_MARKER, inp["marker"] if marker is None else marker)
        for c, t in enumerate((F.TAP_UX, F.TAP_UY, F.TAP_UZ)):
            f.upload_grid(t, inp["u"][c])
        f.upload_grid(F.TAP_P_VEL if which == 0 else F.TAP_P_DEN, inp["p"])
        f.upload_grid(F.TAP_RESIDUAL, inp["rhs"])
        if pos is not None:
            f.set_particles(pos, *(rows or (None, None, None)))

    def run(self, a, b):
        self.f.step_stages(DT, a, b)

    def u(self):
        return [self.f.download_grid(t) for t in (self.F.TAP_UX, self.F.TAP_UY, self.F.TAP_UZ)]

    def residual(self):
        return self.f.download_grid(self.F.TAP_RESIDUAL)

    def marker(self):
        return self.f.download_grid(self.F.TAP_MARKER)

    def particles(self):
        F = self.F
        return self.f.download_particles(F.TAP_POS), [self.f.download_particles(t) for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]


# ------------------------------------------------------------------------------------------------ 1. every stage against the reference
@pytest.mark.gpu
@pytest.mark.parametrize("dims", STEP_SHAPES, ids=[f"{a}x{b}x{c}" for a, b, c in STEP_SHAPES])
def test_stages_match_float64_reference(dims):
    """Stages 1, 4, 5, 7 (with 6's clear), 11, 12 and 13 on salt-and-pepper markers at fills of 3, 50 and 97 %, every element against
    step_ref; every branch of the advection and the correction is taken (summed over the fills)."""
    report = {}
    for fill in FILLS:
        inp = rough_inputs(dims, fill, seed=int(fill * 100) + sum(dims))
        pos, rows = rough_particles(inp, seed=11)
        b = CudaStages(dims, len(pos))
        check_stages(b, inp, pos, rows, STAGES, report=report)
        b.f.close()
    print_report(f"cuda {dims}", report)
    c7, c13 = report[7]["counts"], report[13]["counts"]
    for k, least in (("eaten_x", 2), ("eaten_y", 2), ("eaten_z", 2), ("wall", 10), ("voxel", 5), ("push", 2)):
        assert c7[k] >= least, (k, c7)
    assert c13["wall"] >= 10 and c13["solid"] >= 5, c13


@pytest.mark.gpu
def test_stages_match_float64_reference_without_a_solid_volume():
    """The same without a solid volume (the kernels' vox == nullptr branches: no eaten particles, no voxel test, no push)."""
    dims = (56, 40, 24)
    inp = rough_inputs(dims, 0.5, seed=77, with_vox=False)
    pos, rows = rough_particles(inp, seed=12)
    b = CudaStages(dims, len(pos))
    report = check_stages(b, inp, pos, rows, STAGES)
    b.f.close()
    print_report(f"cuda {dims} no volume", report)
    assert report[7]["counts"]["wall"] >= 10 and report[13]["counts"]["solid"] >= 5


@pytest.mark.gpu
@pytest.mark.parametrize("scatter", [True, False], ids=["scatter", "gather"])
@pytest.mark.parametrize("dims", [(56, 40, 24), (264, 8, 8), (120, 16, 24)], ids=["56x40x24", "264x8x8", "120x16x24"])
def test_projection_and_position_change_visit_the_cells_around_particles_in_solids(dims, scatter):
    """With a solid volume, stage 4 also visits the cells within two cells and stage 11 those within one cell of a non-FLUID cell that holds a
    particle (DESIGN section 3.3), found from the particle words of the last marker pass.  Particles are put into such cells on both sides of
    every 32-cell word edge (x = 32 k - 2 .. 32 k + 1, so that the dilation carries one and two cells across the edge both ways) and next to
    the last x wall; stage 0 (either transfer path's marker pass) records them, then stages 4 and 11 run on the rough inputs of a 3 % fill.
    Every element is compared with step_ref, unwritten ones bit for bit: a region too small leaves random input bits where the reference
    writes, a region too large overwrites input bits the reference keeps."""
    inp = rough_inputs(dims, 0.03, seed=sum(dims) + 1)
    m = inp["marker"]
    nx, ny, nz = dims
    rng = np.random.default_rng(8)
    xs = [x for e in range(32, nx - 1, 32) for x in (e - 2, e - 1, e, e + 1) if 1 <= x <= nx - 2] + [nx - 2]
    cells = []
    for x in xs:
        yz = np.argwhere(m[1:-1, 1:-1, x] != R.FLUID) + 1
        for z, y in yz[rng.choice(len(yz), min(len(yz), 6), replace=False)]:
            cells.append((x, y, z))
    cells = np.array(cells)
    stray = np.zeros(m.shape, dtype=bool)
    stray[cells[:, 2], cells[:, 1], cells[:, 0]] = True
    pos = np.c_[cells + 0.5, np.zeros(len(cells))].astype(np.float32)
    b = CudaStages(dims, len(pos), scatter)
    b.put(inp, 0, pos)
    b.run(0, 1)  # the marker pass of P2G writes the particle words
    extra = R.visited(m, stray, 2) & ~R.near_fluid(m)
    edge = extra[..., 30:34].sum() if nx > 32 else 0
    assert extra.sum() > 100 and edge > 0, (int(extra.sum()), int(edge))
    for st, ref in ((4, R.project(m, inp["u"], inp["p"], inp["vox"], stray=stray)), (11, R.position_change(m, inp["u"], inp["p"], DT, stray=stray))):
        b.put(inp, 0 if st == 4 else 1)
        b.run(st, st + 1)
        for c, got in enumerate(b.u()):
            R.check_grid(got, ref[c], f"stage {st} u[{c}] {dims}")
            assert (ref[c]["written"] & ~R.near_fluid(m)).sum() > 0
    b.f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["dam_small", "sphere"])
def test_stages_match_float64_reference_on_oracle_seeded_inputs(scene):
    """Realistic inputs: one step of dam_small (random APIC rows) or of the 56 x 40 x 24 shapes row with its moving sphere, seeded from the
    oracle at every stage as tests/stagewise.py does -- before each of stages 1, 4, 5, 7, 11, 12 and 13 the oracle's state is handed to a
    fresh CUDA fluid through the taps, the stage runs there and every element is compared with step_ref; then the oracle runs the stage."""
    from oracle import oracle as O
    from tests import util

    if scene == "dam_small":
        orc, dims, vox = util.oracle_from_scene("dam_small"), (32, 32, 32), None
    else:
        dims = (56, 40, 24)
        lo, hi = fluid_box(dims)
        orc = O.OracleFluid(*dims, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
        orc.add_fluid_cube(lo, hi)
        vox = np.asarray(sphere_volume(dims), dtype=np.float16)
        orc.set_voxels(vox.astype(np.float32))
    orc.set_rebin_frequency(0)
    orc.set_gravity_grid([0.0, -981.0, 0.0])
    rng = np.random.default_rng(5)
    orc.set_particles(orc.particles().copy(), *[rng.normal(0, 3.0, (orc.num_particles, 4)).astype(np.float32) for _ in range(3)])
    orc.step_stages(DT, 0, 1)
    report = {}
    for st in range(1, 14):
        if st == 6:
            continue  # checked with 7 (the clear and the advection)
        if st in STAGES:
            u = [orc.grid(a).copy() for a in (O.ARR_UX, O.ARR_UY, O.ARR_UZ)]
            inp = {"dims": dims, "marker": orc.grid(O.ARR_MARKER).copy(), "u": u, "disp": u, "vox": vox,
                   "p": orc.grid(O.ARR_P_VEL if st < 10 else O.ARR_P_DEN).copy(), "rhs": orc.grid(O.ARR_RESIDUAL).copy()}
            pos = orc.particles().copy()
            pos[:, 3] = 0.0
            rows = [orc.particles(a).copy() for a in (O.ARR_ROWX, O.ARR_ROWY, O.ARR_ROWZ)]
            b = CudaStages(dims, len(pos))
            check_stages(b, inp, pos, rows, [st], report=report)
            b.f.close()
        orc.step_stages(DT, 6 if st == 7 else st, st + 1)
    print_report(f"oracle-seeded {scene}", report)
    if vox is not None:
        c7 = report[7]["counts"]
        assert c7["eaten_x"] + c7["eaten_y"] + c7["eaten_z"] >= 10 and c7["hit"] >= 10, c7


# ------------------------------------------------------------------------------------------------ 2. particle counts around the grid-stride size
def _stride_size():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 128 * 256  # particle_blocks(): min(blocks, SMs x 128) blocks of 256


@pytest.mark.gpu
def test_particle_counts_around_the_grid_stride_size():
    """size - 1, size and size + 37 particles (size = SMs x 128 x 256 threads; + 37: a partial last warp in the second pass): the full
    count checked element by element for the advection and the correction (in chunks), the common prefix of the other counts bit for bit."""
    dims = (48, 48, 8)
    size = _stride_size()
    inp = rough_inputs(dims, 0.5, seed=5)
    rng = np.random.default_rng(6)
    fl = np.argwhere(inp["marker"] == R.FLUID)[:, ::-1]
    n = size + 37
    pos = np.c_[fl[rng.integers(0, len(fl), n)] + rng.random((n, 3)), rng.uniform(-1, 1, n)].astype(np.float32)
    rows = [rng.normal(0, 10.0, (n, 4)).astype(np.float32) for _ in range(3)]
    outs = {}
    for count in (size + 37, size, size - 1):
        b = CudaStages(dims, count)
        b.put(inp, 0, pos[:count], [r[:count] for r in rows])
        b.run(6, 8)
        adv = b.particles()
        b.put(dict(inp, u=inp["disp"]), 1, pos[:count], [r[:count] for r in rows])
        b.run(13, 14)
        outs[count] = (adv, b.particles()[0])
        b.f.close()
    (ap, ar), cp = outs[size + 37]
    chunk = 1 << 20
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        ref = R.advect(inp["u"], inp["vox"], pos[s:e], DT)
        R.check_particles(ap[s:e], ref, f"advection, particles {s}..{e}", got_rows=[r[s:e] for r in ar])
        ref = R.correct(inp["disp"], inp["marker"], pos[s:e])
        R.check_particles(cp[s:e], ref, f"correction, particles {s}..{e}")
    for count in (size, size - 1):
        (bp, br), bc = outs[count]
        assert np.array_equal(bp.view(np.uint32), ap[:count].view(np.uint32)), count
        assert all(np.array_equal(x.view(np.uint32), y[:count].view(np.uint32)) for x, y in zip(br, ar)), count
        assert np.array_equal(bc.view(np.uint32), cp[:count].view(np.uint32)), count


# ------------------------------------------------------------------------------------------------ 3. stale faces are never read (B6)
POISON_SCENES = ["shape", "dam_small"]


def _fluid(scene, scatter, graph, solid):
    """A fluid of the scene (the 56 x 40 x 24 row's box fluid, or dam_small), optionally with a moving solid that starts inside the fluid (the
    shapes row's rigid sphere; in dam_small a moving slab through the dam), returning (fluid, the kept solid volume)."""
    import torch
    import blub_b200
    from tests import util

    if scene == "shape":
        dims = (56, 40, 24)
        lo, hi = fluid_box(dims)
        f = blub_b200.HybridFluid(*dims, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
        f.add_fluid_cube(lo, hi)
        vol = sphere_volume(dims) if solid else None
    else:
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
        vol = None
        if solid:
            vol = np.zeros((32, 32, 32, 4), dtype=np.float16)
            vol[4:28, 1:12, 16:19] = (5.0, 1.0, -2.0, 1.0)
    f.set_gravity_grid([0.0, -981.0, 0.0])
    f.set_transfer_path(scatter)
    f.set_graph_replay(graph)
    keep = None
    if vol is not None:
        keep = torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float16)).to("cuda")
        torch.cuda.synchronize()
        f.set_solid_voxels(keep.data_ptr())
    return f, keep


def _state(f):
    from blub_b200 import fluid as F

    f.synchronize()
    m = f.download_grid(F.TAP_MARKER)
    grids = {t: f.download_grid(getattr(F, t)) for t in ("TAP_UX", "TAP_UY", "TAP_UZ", "TAP_P_VEL", "TAP_P_DEN", "TAP_RESIDUAL")}
    parts = {t: f.download_particles(getattr(F, t)) for t in ("TAP_POS", "TAP_VX", "TAP_VY", "TAP_VZ")}
    return m, grids, parts, [f.last_solve(w) for w in (0, 1)]


def _same(a, b, what, faces=None, taps=("TAP_P_VEL", "TAP_P_DEN", "TAP_RESIDUAL")):
    """Particles, rows, marker, the pressures / residual `taps` on FLUID cells, the faces `faces` (c -> mask) and the solver statistics
    of the poisoned fluid bit for bit those of its twin, and finite."""
    ma, ga, pa, sa = a
    mb, gb, pb, sb = b
    assert np.array_equal(ma, mb), f"{what}: marker"
    fl = ma == R.FLUID
    for t in pa:
        assert np.isfinite(pa[t]).all() and np.array_equal(pa[t].view(np.uint32), pb[t].view(np.uint32)), f"{what}: {t}"
    for t in taps:
        x, y = ga[t][fl], gb[t][fl]
        assert np.isfinite(x).all() and np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"{what}: {t} on FLUID cells"
    for c, t in enumerate(("TAP_UX", "TAP_UY", "TAP_UZ")):
        sel = R.near_fluid(ma) if faces is None else faces[c]
        x, y = ga[t][sel], gb[t][sel]
        bad = ~np.isfinite(x) | (x.view(np.uint32) != y.view(np.uint32))
        assert not bad.any(), f"{what}: {t}: {int(bad.sum())} faces differ, first at [z, y, x] = {tuple(np.argwhere(sel)[np.argmax(bad)])}"
    assert sa == sb, f"{what}: solver statistics {sa} vs {sb}"


def _stray(m, pos, solid):
    """Non-FLUID cells that hold a particle (positions clamped to [1, n - 1], as the marker passes do), with a solid volume; else None."""
    if not solid:
        return None
    S = np.array([m.shape[2], m.shape[1], m.shape[0]])
    c = np.minimum(np.clip(pos[:, :3], 1.0, S - 1.0).astype(np.int64), S - 1)
    out = np.zeros(m.shape, dtype=bool)
    out[c[:, 2], c[:, 1], c[:, 0]] = True
    return out & (m != R.FLUID)


def _eaten(f, keep):
    """Particles whose cell has a solid voxel with w > 0 (advect_kernel_one moves them one cell before G2P)."""
    if keep is None:
        return 0
    from blub_b200 import fluid as F

    w = keep.float().cpu().numpy()[..., 3]
    p = f.download_particles(F.TAP_POS)[:, :3]
    S = np.array([w.shape[2], w.shape[1], w.shape[0]])
    c = np.clip(np.floor(p).astype(np.int64), 0, S - 1)
    return int((w[c[:, 2], c[:, 1], c[:, 0]] > 0).sum())


def _poison_u(f, poison):
    from blub_b200 import fluid as F

    for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ):
        g = f.download_grid(t)
        f.upload_grid(t, np.full_like(g, np.nan) if poison else g)


@pytest.mark.gpu
@pytest.mark.parametrize("solid", [False, True], ids=["open", "moving_solid"])
@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("scatter", [True, False], ids=["scatter", "gather"])
@pytest.mark.parametrize("scene", POISON_SCENES)
def test_poisoned_faces_are_never_read_in_full_steps(scene, scatter, graph, solid):
    """16 steps; before every step every velocity face of one fluid is set to NaN, its twin makes the same download / upload round trip with
    its own values.  After every step both agree bit for bit (module _same, faces within one cell of FLUID) and are finite."""
    a, ka = _fluid(scene, scatter, graph, solid)
    b, kb = _fluid(scene, scatter, graph, solid)
    eaten = 0
    for k in range(16):
        eaten += _eaten(a, ka)
        _poison_u(a, True)
        _poison_u(b, False)
        a.step(DT)
        b.step(DT)
        sa = _state(a)
        # the faces the next step's P2G leaves to the correction's reads: those within one cell of FLUID (the cells around particles in
        # solids are checked stage by stage below, where the particles the marker passes recorded are known)
        _same(sa, _state(b), f"{scene} step {k}", _read_faces(sa[0], 12))
    print(f"{scene} eaten particles over 16 steps: {eaten}")
    assert eaten >= (20 if solid else 0), eaten  # the moving solid swallows particles: the path the region rule is about is taken
    a.close()
    b.close()
    del ka, kb


def _read_faces(m, stage, stray=None):
    """The faces the stages after `stage` read, for component c (DESIGN section 3.3): after P2G (0 .. 3) the divergence reads the faces of
    FLUID cells and their -c neighbours; after the projection (4 .. 10) G2P reads the cells within one cell of FLUID and, with a solid volume,
    an eaten particle those within two cells of its non-FLUID cell (stray); after the position change (11 .. 13) the correction reads the
    cells within one cell of FLUID and of a non-FLUID cell that holds a particle."""
    if stage <= 3:
        fl = m == R.FLUID
        return [fl | R.shift(fl, R.unit(c), False) for c in range(3)]
    return [R.visited(m, stray, 2 if stage <= 10 else 1)] * 3


@pytest.mark.gpu
@pytest.mark.parametrize("solid", [False, True], ids=["open", "moving_solid"])
@pytest.mark.parametrize("scatter", [True, False], ids=["scatter", "gather"])
@pytest.mark.parametrize("scene", POISON_SCENES)
def test_poisoned_faces_and_pressures_are_never_read_stage_by_stage(scene, scatter, solid):
    """Six steps stage by stage (eager): the velocity faces are poisoned before stage 0, the pressure of each solve and the residual on every
    non-FLUID cell before stages 2 and 10; the twin makes the same round trips.  After every stage both agree bit for bit."""
    from blub_b200 import fluid as F

    a, ka = _fluid(scene, scatter, False, solid)
    b, kb = _fluid(scene, scatter, False, solid)
    eaten = 0
    for k in range(6):
        eaten += _eaten(a, ka)
        for st in range(14):
            if st in (0, 8):  # the particles the marker pass of this stage records
                stray_pos = a.download_particles(F.TAP_POS) if st == 0 else None
            for f, poison in ((a, True), (b, False)):
                if st == 0:
                    _poison_u(f, poison)
                if st in (2, 10):
                    m = f.download_grid(F.TAP_MARKER)
                    for t in (F.TAP_P_VEL if st == 2 else F.TAP_P_DEN, F.TAP_RESIDUAL):
                        g = f.download_grid(t)
                        if poison:
                            g[m != R.FLUID] = np.nan
                        f.upload_grid(t, g)
                f.step_stages(DT, st, st + 1)
            sa, sb = _state(a), _state(b)
            if st == 8:
                stray_pos = sa[2]["TAP_POS"]  # the advected particles: the ones stage 8's marker pass records
            if st in (6, 7, 8, 9, 10):  # the faces the next grid pass or particle stage reads: those of the marker stage 4 saw
                faces = _read_faces(m_before, 5, stray_before)
            else:
                m_before = sa[0]
                stray_before = _stray(m_before, stray_pos, solid)
                faces = _read_faces(m_before, st, stray_before)
            # the pressure / residual the stage wrote on the marker's FLUID cells (the poisoned values stay on cells no stage rewrote yet)
            taps = {1: ("TAP_RESIDUAL",), 9: ("TAP_RESIDUAL",)}.get(st, ("TAP_P_VEL", "TAP_RESIDUAL") if 2 <= st <= 5 else
                                                                        (("TAP_P_DEN", "TAP_RESIDUAL") if st >= 10 else ()))
            _same(sa, sb, f"{scene} step {k} stage {st}", faces, taps)
    print(f"{scene} eaten particles over 6 steps: {eaten}")
    assert eaten >= (10 if solid else 0), eaten
    a.close()
    b.close()
    del ka, kb
