"""The stage-by-stage comparison of one fluid step, shared by the small-scene and the BASELINE-config parity tests.

Both implementations walk the 14 stages of HybridFluid::step (hybrid_fluid.rs:770-977) from identical particles; after every stage the taps
are compared (SURVEY.md section 8c tolerances) and the CUDA side is re-seeded from the oracle's output, so that every stage is judged on
IDENTICAL inputs and round-off does not leak from one stage into the next.
"""
import numpy as np

from blub_b200 import fluid as F
from oracle import oracle as O
from tests import advect_ref, util
from tests.util import DT, grid_close

STAGE_TAPS = [(F.TAP_UX, O.ARR_UX), (F.TAP_UY, O.ARR_UY), (F.TAP_UZ, O.ARR_UZ)]
ROW_TAPS = [(F.TAP_VX, O.ARR_ROWX), (F.TAP_VY, O.ARR_ROWY), (F.TAP_VZ, O.ARR_ROWZ)]


def particles_close(p_o, p_g, what, tol, frac=1.0, loose=None):
    """max|d| <= tol for all particles (frac == 1), or for all but a fraction 1 - frac of them (those within `loose`): a particle that sits
    within round-off of a discontinuous branch of the wall handling (advect_particles.comp:134-173) may take the other branch."""
    d = np.abs(np.asarray(p_o, np.float64) - np.asarray(p_g, np.float64))
    d = d.reshape(d.shape[0], -1).max(axis=1)
    if frac >= 1.0:
        assert d.max() <= tol, f"{what}: max|d| = {d.max():.3e} > {tol:.1e}"
    else:
        q = np.quantile(d, frac)
        assert q <= tol, f"{what}: {frac:.4%} quantile |d| = {q:.3e} > {tol:.1e}"
        if loose is not None:
            assert d.max() <= loose, f"{what}: max|d| = {d.max():.3e} > {loose:.1e}"
    return d.max()


def solve_stage(orc, gpu, which, stage, converged):
    """Stage 2 / 10.  With the scene's solver configuration the iteration counts must agree (stop decisions are taken at every 4th iteration
    on max|r| < tol).  Small scenes (`converged` = False) also compare the iterate itself at that point.  On the BASELINE-size scenes the
    unconverged 32-iteration iterate of an fp32 CG is not a well-conditioned quantity (the two implementations sum their dot products in
    different orders and drift apart by > 1 % of max|p| within 32 iterations at 256 x 128 x 128), so there the SOLUTION is compared: both
    run the same right-hand side to convergence (tolerance 1e-4, SURVEY 8c), the CUDA result must satisfy max|b - A p| < tolerance when the
    residual is recomputed independently in float64, need about as many iterations as the oracle, and agree with the oracle's pressure."""
    tap_p, arr_p = (F.TAP_P_VEL, O.ARR_P_VEL) if which == 0 else (F.TAP_P_DEN, O.ARR_P_DEN)
    rhs = orc.grid(O.ARR_RESIDUAL).copy()
    p0 = orc.grid(arr_p).copy()
    m = orc.grid(O.ARR_MARKER).copy()
    orc.step_stages(DT, stage, stage + 1)
    gpu.step_stages(DT, stage, stage + 1)
    (eo, io), (eg, ig) = orc.last_solve(which), gpu.last_solve(which)
    if not converged:
        assert io == ig, (which, io, ig)
        grid_close(orc.grid(arr_p), gpu.download_grid(tap_p), f"p{which + 1}", rel=5e-3, abs_=1e-4)
        return io
    assert abs(io - ig) <= 4 and ig % 4 == 0, (which, io, ig, eo, eg)
    p_default = orc.grid(arr_p).copy()
    tol = 1e-4
    for f in (orc, gpu):
        f.set_solver_config(which, tol, 4000, 4)
    orc.grid(O.ARR_RESIDUAL)[:] = rhs
    orc.grid(arr_p)[:] = p0
    gpu.upload_grid(F.TAP_RESIDUAL, rhs)
    gpu.upload_grid(tap_p, p0)
    orc.solve(which, DT)
    gpu.solve_only(which, DT)
    (eo, io), (eg, ig) = orc.last_solve(which), gpu.last_solve(which)
    assert 0 < io < 4000 and 0 < ig < 4000 and abs(io - ig) <= 8 + 0.05 * io, (which, io, ig)
    pg = gpu.download_grid(tap_p)
    b64 = np.where(m == O.FLUID, rhs, 0.0)
    res_g = np.abs(b64 - util.apply_A(m, pg)).max()
    res_o = np.abs(b64 - util.apply_A(m, orc.grid(arr_p))).max()
    # the recursive residual of an fp32 CG drifts away from the true one over hundreds of iterations (in the oracle as well): the TRUE
    # residual of the CUDA solution, recomputed in float64, has to be as good as the oracle's
    assert eg < tol / DT and res_g <= 1.25 * max(res_o, tol / DT) + 1e-6 * np.abs(rhs).max(), (eg, res_g, res_o, tol / DT)
    grid_close(orc.grid(arr_p), pg, f"p{which + 1} converged ({io} / {ig} iterations)", rel=5e-3, abs_=1e-3)
    for f in (orc, gpu):
        f.set_solver_config(which, 0.1, 32, 4)
    orc.grid(arr_p)[:] = p_default  # continue from the default solve's pressure
    return io


def flipped_particles(p_o, p_g, x1, near, what, tol, max_flips=2):
    """Non-robust particle comparison with a solid volume: max|d| <= tol for every particle except those whose float64-restated end point x1
    lies within round-off of a cell plane or a clamp plane (tests/advect_ref.py) -- nvcc contracts FMAs, the oracle does not, so such a
    particle may take the other hit / push branch.  At most `max_flips` of them; they are printed.  Returns the mask of flipped particles."""
    d = np.abs(np.asarray(p_o, np.float64) - np.asarray(p_g, np.float64))
    d = d.reshape(d.shape[0], -1).max(axis=1)
    bad = d > tol
    for i in np.nonzero(bad)[0]:
        print(f"{what}: particle {i} took another branch: oracle {p_o[i]}, CUDA {p_g[i]}, restated x1 {x1[i]}, on a plane: {bool(near[i])}")
    assert not (bad & ~near).any(), f"{what}: max|d| = {d[~near].max():.3e} > {tol:.1e} away from every cell and clamp plane"
    assert bad.sum() <= max_flips, f"{what}: {int(bad.sum())} particles on a plane took another branch"
    return bad


def compare_one_step(orc, gpu, robust=False, vox=None, min_contact=(1, 1)):
    """robust = True: the big-scene form (fixed-iteration iterate comparison, quantile-based particle checks).
    vox: the solid volume of this step as float32 [nz, ny, nx, 4] (the fp16 values the GPU reads).  The oracle gets it; after stage 0 the volume
    the CUDA step reads (borrowed or composed with floating bodies) must equal it bit for bit; the fluid must touch the solid (util.solid_contact
    >= min_contact at the start of the step and after advection); particle comparisons stay max-error comparisons, with at most two particles
    allowed another branch, each within round-off of a plane.  The solves are compared by their converged solutions there (as on the big
    scenes): next to moving solids the 32-iteration iterate of the density solve is not a well-conditioned quantity, and every later stage starts
    from the oracle's pressure anyway."""
    run = lambda a, b: (orc.step_stages(DT, a, b), gpu.step_stages(DT, a, b))
    npart = orc.num_particles
    frac = 0.9999 if robust else 1.0
    converged = robust or vox is not None
    report = {}
    if vox is not None:
        assert not robust
        vox = np.ascontiguousarray(vox, dtype=np.float32)
        orc.set_voxels(vox)
    run(0, 1)  # P2G
    m_o, m_g = orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER)
    assert np.array_equal(m_o, m_g)
    if vox is not None:
        assert np.array_equal(gpu.download_solid_voxels().astype(np.float32).view(np.uint32), vox.view(np.uint32))
        report["contact0"] = util.solid_contact(m_o, vox, orc.particles())
        assert all(c >= lo for c, lo in zip(report["contact0"], min_contact)), (report["contact0"], min_contact)
    for c, (tg, to) in enumerate(STAGE_TAPS):
        report[f"p2g{c}"] = grid_close(orc.grid(to), gpu.download_grid(tg), f"P2G u[{c}]", mask=util.fluid_adjacent_faces(m_o, c))
    fl = m_o == O.FLUID
    run(1, 2)  # rhs 1
    report["rhs1"] = grid_close(orc.grid(O.ARR_RESIDUAL), gpu.download_grid(F.TAP_RESIDUAL), "rhs1", mask=fl)
    gpu.upload_grid(F.TAP_RESIDUAL, orc.grid(O.ARR_RESIDUAL))
    report["iterations1"] = solve_stage(orc, gpu, 0, 2, converged)
    # continue from the ORACLE's pressure so that solver round-off does not leak into the per-stage comparison
    gpu.upload_grid(F.TAP_P_VEL, orc.grid(O.ARR_P_VEL))
    near = util.near_fluid(m_o)  # the grid passes visit the cells within one cell of the fluid (see util.near_fluid)
    run(3, 5)  # (binning off) + divergence_remove
    for c, (tg, to) in enumerate(STAGE_TAPS):
        grid_close(orc.grid(to), gpu.download_grid(tg), f"projected u[{c}]", mask=near)
    run(5, 6)  # extrapolate
    for c, (tg, to) in enumerate(STAGE_TAPS):
        grid_close(orc.grid(to), gpu.download_grid(tg), f"extrapolated u[{c}]", mask=near)
    for c, (tg, to) in enumerate(STAGE_TAPS):
        gpu.upload_grid(tg, orc.grid(to))
    if vox is not None:
        branches = advect_ref.advect([orc.grid(to) for _, to in STAGE_TAPS], vox, orc.particles(), DT)
    run(6, 9)  # clear + advect + boundary marker
    p_o = orc.particles()[:, :3]
    vmax = max(max(np.abs(orc.particles(to)[:, 3]).max() for _, to in ROW_TAPS), 1.0)
    if vox is None:
        assert np.array_equal(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER)) if not robust else util.markers_agree(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER)) >= 0
        report["advect"] = particles_close(p_o, gpu.download_particles()[:, :3], "advected positions", 2e-4, frac, loose=0.5)
        for k, (tg, to) in enumerate(ROW_TAPS):
            particles_close(orc.particles(to), gpu.download_particles(tg), f"APIC row {k}", 1e-3 * vmax, frac, loose=None)
    else:
        p_g = gpu.download_particles()[:, :3]
        flips = flipped_particles(p_o, p_g, branches["x1"], branches["near_plane"], "advected positions", 2e-4)
        keep = ~flips
        report["advect"] = particles_close(p_o[keep], p_g[keep], "advected positions", 2e-4)
        report["advect_flips"] = int(flips.sum())
        for k, (tg, to) in enumerate(ROW_TAPS):
            particles_close(orc.particles(to)[keep], gpu.download_particles(tg)[keep], f"APIC row {k}", 1e-3 * vmax)
        m_o, m_g = orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER)
        # a flipped particle may mark another cell FLUID; every other cell agrees
        own = np.zeros(m_o.shape, dtype=bool)
        for p in (p_o[flips], p_g[flips]):
            c = np.floor(p).astype(np.int64)
            own[c[:, 2], c[:, 1], c[:, 0]] = True
        assert not ((m_o != m_g) & ~own).any(), "marker after advection"
        report["contact7"] = util.solid_contact(m_o, vox, p_o)
        assert all(c >= lo for c, lo in zip(report["contact7"], min_contact)), (report["contact7"], min_contact)
        report["branches"] = {k: int(branches[k].sum()) for k in ("eaten", "wall", "voxel", "push")}
        report["advect_ref"] = branches
    gpu.set_particles(np.c_[p_o, np.zeros(npart, np.float32)], orc.particles(O.ARR_ROWX), orc.particles(O.ARR_ROWY), orc.particles(O.ARR_ROWZ))
    gpu.upload_grid(F.TAP_MARKER, orc.grid(O.ARR_MARKER))
    run(9, 10)  # rhs 2
    fl = orc.grid(O.ARR_MARKER) == O.FLUID
    report["rhs2"] = grid_close(orc.grid(O.ARR_RESIDUAL), gpu.download_grid(F.TAP_RESIDUAL), "rhs2", rel=1e-4, abs_=2e-3, mask=fl)
    gpu.upload_grid(F.TAP_RESIDUAL, orc.grid(O.ARR_RESIDUAL))
    report["iterations2"] = solve_stage(orc, gpu, 1, 10, converged)
    gpu.upload_grid(F.TAP_P_DEN, orc.grid(O.ARR_P_DEN))
    near = util.near_fluid(orc.grid(O.ARR_MARKER))
    run(11, 13)  # position change + extrapolate
    for c, (tg, to) in enumerate(STAGE_TAPS):
        grid_close(orc.grid(to), gpu.download_grid(tg), f"displacement[{c}]", mask=near)
        gpu.upload_grid(tg, orc.grid(to))
    if vox is not None:
        corr = advect_ref.correct([orc.grid(to) for _, to in STAGE_TAPS], orc.grid(O.ARR_MARKER), orc.particles())
    run(13, 14)  # correct particles
    if vox is None:
        report["correct"] = particles_close(orc.particles()[:, :3], gpu.download_particles()[:, :3], "corrected positions", 2e-4, frac, loose=0.5)
    else:
        p_o, p_g = orc.particles()[:, :3], gpu.download_particles()[:, :3]
        flips = flipped_particles(p_o, p_g, corr["x1"], corr["near_plane"], "corrected positions", 2e-4)
        report["correct"] = particles_close(p_o[~flips], p_g[~flips], "corrected positions", 2e-4)
        report["correct_flips"] = int(flips.sum())
        report["correct_hits"] = {k: int(corr[k].sum()) for k in ("wall", "marker")}
        report["correct_ref"] = corr
    return report
