"""Float64 restatements of the grid passes, the advection and the density correction of the fluid step (fluid_kernels.cu), with a bound
for every element they round, the elements they must reproduce bit for bit, and both branches of every decision a particle takes within
its own rounding bound.  NumPy only; independent of the oracle.  Volumes are [z, y, x]; positions (x, y, z); component c lies along axis
2 - c of a volume.

What is exact (compared bit for bit):
  * every element a stage does not write keeps its input bits: divergence_compute (stage 1) writes FLUID cells only; divergence_remove
    (4) and position_change (11) write the cells within one cell (26-neighbourhood) of a FLUID cell and, with a solid volume, those within
    two (4) / one (11) cells of a non-FLUID cell that holds a particle (`stray`: the faces an eaten or pushed particle reads); the
    extrapolation (5, 12) writes the invalid faces that have a valid in-plane neighbour;
  * stage 4's faces with a SOLID side take the fp16 voxel value of the SOLID cell (0 past the grid's last cell), faces without a FLUID
    side 0; stage 11's faces with a SOLID side 0;
  * the float32 position arithmetic the kernels do on the particles' own coordinates: x0 +- 1 (the eaten shift), max(0, x0 - off),
    the truncations, floor and fract of those values.  For float32 inputs every one of them is a single correctly rounded operation, which
    NumPy's float32 arithmetic reproduces exactly, so the corner indices and the G2P / correction fractions are the kernels' own;
  * the advection's marker: the cells that hold an advected particle are FLUID, every other cell is AIR (after stage 6's clear).

The bounds.  Every other output is followed through the kernel's float32 operations as a pair (value, error bound): the value in float64,
the bound propagated to first order with u = 2^-24 per rounding times the magnitude of the rounded result,
    a +- b: e_a + e_b + u |a +- b|        a b: |b| e_a + |a| e_b + u |a b|        a / b: (e_a + |a / b| e_b) / |b| + u |a / b|
    sqrt(a): e_a / (2 sqrt(a)) + u sqrt(a)        saturate, fmin, fmax, clamp: 1-Lipschitz (fmin / fmax: the largest error among the
    operands that can be the extreme one).
A contracted FMA a b + c rounds once where the separate operations round twice, and the first rounding's term u |a b| is part of the sum
above: the bound holds with nvcc's contraction and without it (the oracle is built with -ffp-contract=off).  mix(a, b, t) =
a (1 - t) + b t is three products / sums and 1 - t; float constants (1/6, 1e-10, 0.001, 1.001) enter as their float32 values.  The
push's voxel_w_trilinear at x1 +- e_k takes its fraction from a rounded position: a trilinear sample is continuous and moves by at most
(w_max - w_min) per unit of fraction along each axis, whichever cell the floor picks, so its error is that spread times the sum of the
three fraction errors plus its own roundings.  Every bound is multiplied by 1.001 (second-order terms) and 1e-30 is added (denormals).

Decisions.  Where a particle's float64 value lies within its own bound of a decision -- a clamp plane 1.001f / n - 1.001f, a cell plane
for the voxel, SOLID, same-cell and marker tests, the sign of a component that picks fract or 1 - fract -- the kernel may decide either
way.  The reference then evaluates every combination of those decisions (advect: hit, same cell, the three signs; correct: hit, the
three signs) and the kernel has to match one of these branches within that branch's bounds; the marker cell of such a particle may be
any cell its end point can round into.
"""
import itertools

import numpy as np

SOLID, FLUID, AIR = 0, 1, -1
U = 2.0 ** -24
SAFETY = 1.001
TINY = 1e-30
f32 = np.float32


# ------------------------------------------------------------------------------------------------ (value, bound) arithmetic
class E:
    """A float64 value with a first-order bound on the error of the kernel's float32 result (module docstring)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, dtype=np.float64)

    def __add__(self, o):
        o = _e(o)
        v = self.v + o.v
        return E(v, self.e + o.e + U * np.abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = _e(o)
        v = self.v - o.v
        return E(v, self.e + o.e + U * np.abs(v))

    def __rsub__(self, o):
        return _e(o) - self

    def __mul__(self, o):
        o = _e(o)
        v = self.v * o.v
        return E(v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + U * np.abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _e(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            e = (self.e + np.abs(v) * o.e) / np.abs(o.v) + U * np.abs(v)
        return E(v, e)

    def __getitem__(self, k):
        return E(self.v[k], self.e[k])


def _e(x):
    return x if isinstance(x, E) else E(x)


def mix(a, b, t):
    """mixf(a, b, t) = a (1 - t) + b t."""
    return _e(a) * (1.0 - _e(t)) + _e(b) * _e(t)


def sat(a):
    return E(np.clip(a.v, 0.0, 1.0), a.e)


def sqrt(a):
    v = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(v > 0.0, a.e / (2.0 * v), np.sqrt(a.e)) + U * v
    return E(v, e)


def fmin(*xs):
    """fminf over the operands; the bound is the largest among those operands that can be the minimum."""
    xs = [_e(x) for x in xs]
    v = np.minimum.reduce([x.v for x in xs])
    k = np.argmin([x.v for x in xs], axis=0)
    em = np.choose(k, [x.e for x in xs])
    e = np.zeros_like(v)
    for x in xs:
        with np.errstate(invalid="ignore"):
            can = x.v - x.e <= v + em
        e = np.where(can, np.maximum(e, x.e), e)
    return E(v, e)


def clampv(a, lo, hi):
    return E(np.minimum(np.maximum(a.v, lo), hi), a.e)


def bound(e):
    return SAFETY * e + TINY


# ------------------------------------------------------------------------------------------------ grid helpers
def shift(a, d, fill):
    """a at (x + d[0], y + d[1], z + d[2]) for every cell (x, y, z); `fill` past the grid."""
    out = np.full_like(a, fill)
    src, dst = [], []
    for ax, k in zip((2, 1, 0), d):
        n = a.shape[ax]
        if k >= 0:
            src.append(slice(k, n)), dst.append(slice(0, n - k))
        else:
            src.append(slice(0, n + k)), dst.append(slice(-k, n))
    s = [None] * 3
    t = [None] * 3
    for ax, sl, dl in zip((2, 1, 0), src, dst):
        s[ax], t[ax] = sl, dl
    out[tuple(t)] = a[tuple(s)]
    return out


def unit(c, k=1):
    d = [0, 0, 0]
    d[c] = k
    return d


def dilate(mask, r):
    """Cells within r cells (Chebyshev) of a set cell."""
    out = np.zeros_like(mask)
    for d in itertools.product(range(-r, r + 1), repeat=3):
        out |= shift(mask, d, False)
    return out


def visited(m, stray, r):
    """The cells stages 4 (r = 2) and 11 (r = 1) visit: within one cell of FLUID, and within r cells of a non-FLUID cell that holds a
    particle (stray: the cells the last marker pass found particles in, with a solid volume; None: none).  After a marker pass such a cell
    is SOLID; the kernels take the particle words minus the FLUID bits of the marker they see."""
    out = near_fluid(m)
    return out if stray is None else out | dilate(np.asarray(stray, dtype=bool) & (np.asarray(m) != FLUID), r)


def near_fluid(m):
    """Cells within one cell (26-neighbourhood) of a FLUID cell: the cells stages 4 and 11 visit."""
    fl = np.asarray(m) == FLUID
    out = np.zeros_like(fl)
    for d in itertools.product((-1, 0, 1), repeat=3):
        out |= shift(fl, d, False)
    return out


def valid_faces(m, c):
    """Faces of component c whose cell or +c neighbour is FLUID (extrapolate_velocity.comp:5-10)."""
    fl = np.asarray(m) == FLUID
    return fl | shift(fl, unit(c), False)


def voxel_values(vox, shape):
    """The float32 values of the fp16 solid volume [nz, ny, nx, 4] (zeros without one)."""
    if vox is None:
        return np.zeros(shape + (4,), dtype=np.float32)
    return np.asarray(vox, dtype=np.float16).astype(np.float32)


def grid_out(inp, written, exact, exact_value, value):
    """One output grid: written & exact -> exact_value (bit for bit), written & ~exact -> value (an E), not written -> the input's bits."""
    inp = np.asarray(inp, dtype=np.float32)
    bits = np.where(written & exact, np.asarray(exact_value, dtype=np.float32), inp)
    rounded = written & ~exact
    want = np.where(rounded, value.v, np.nan)
    return {"bits": bits, "exact": ~rounded, "written": written, "want": want, "bound": np.where(rounded, bound(value.e), 0.0)}


def check_grid(got, out, what, unwritten=True):
    """The kernel's grid against one output of a stage function: exact elements bit for bit (with unwritten = False only the written ones:
    the oracle writes every cell), rounded ones within their bounds.  Returns err / bound of the rounded elements."""
    got = np.asarray(got, dtype=np.float32)
    ex = out["exact"] if unwritten else (out["exact"] & out["written"])
    badx = ex & (got.view(np.uint32) != out["bits"].view(np.uint32))
    if badx.any():
        k = tuple(int(i) for i in np.argwhere(badx)[0])
        raise AssertionError(f"{what}: {int(badx.sum())} exact elements differ; first at [z, y, x] = {k}: got {got[k]!r}, want {out['bits'][k]!r}"
                             f" ({'written' if out['written'][k] else 'not written: the input'})")
    r = ~out["exact"]
    err = np.abs(got[r].astype(np.float64) - out["want"][r])
    b = out["bound"][r]
    bad = ~(err <= b)
    if bad.any():
        j = int(np.argmax(np.where(bad, np.nan_to_num(err - b, nan=np.inf), -np.inf)))
        k = tuple(int(i) for i in np.argwhere(r)[j])
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(r.sum())} rounded elements beyond their bound; worst at [z, y, x] = {k}: "
                             f"got {got[k]!r}, float64 {out['want'][k]!r}, bound {b[j]:.3e}")
    return np.where(err > 0.0, err / b, 0.0)


# ------------------------------------------------------------------------------------------------ stage 1: divergence
def divergence(m, u, vox, rhs_in):
    """divergence_compute_kernel: on FLUID cells d = sum_c (u_c - u_c(-c)) + the six solid terms, in the kernel's order."""
    m = np.asarray(m)
    vv = voxel_values(vox, m.shape)
    u = [np.asarray(a, dtype=np.float32) for a in u]
    p = [E(u[c]) for c in range(3)]
    n = [E(shift(u[c], unit(c, -1), 0.0)) for c in range(3)]
    d = p[0] - n[0]
    d = d + (p[1] - n[1])
    d = d + (p[2] - n[2])
    for c in range(3):  # -x, -y, -z
        s = shift(m, unit(c, -1), AIR) == SOLID
        t = d + (n[c] - E(shift(vv[..., c], unit(c, -1), 0.0)))
        d = E(np.where(s, t.v, d.v), np.where(s, t.e, d.e))
    for c in range(3):  # +x, +y, +z
        s = shift(m, unit(c), AIR) == SOLID
        t = d - (p[c] - E(shift(vv[..., c], unit(c), 0.0)))
        d = E(np.where(s, t.v, d.v), np.where(s, t.e, d.e))
    fl = m == FLUID
    return grid_out(rhs_in, fl, np.zeros_like(fl), 0.0, d)


# ------------------------------------------------------------------------------------------------ stages 4 and 11
def _face_sides(m, c):
    mc = np.asarray(m)
    mn = shift(mc, unit(c), SOLID)  # past the last cell: SOLID
    inb = shift(np.ones(mc.shape, dtype=bool), unit(c), False)
    return mc, mn, inb


def project(m, u, p, vox, stray=None):
    """divergence_remove_kernel on the cells within one cell of FLUID: faces with a FLUID side take the SOLID cell's voxel (this cell's
    first, 0 past the grid) or u - (p_c - p_n) with p = 0 off FLUID; faces without a FLUID side 0."""
    m = np.asarray(m)
    vv = voxel_values(vox, m.shape)
    p = np.asarray(p, dtype=np.float32)
    near = visited(m, stray, 2)
    out = []
    for c in range(3):
        mc, mn, inb = _face_sides(m, c)
        pc = np.where(mc == FLUID, p, 0.0)
        pn = np.where(mn == FLUID, shift(p, unit(c), 0.0), 0.0)
        val = E(u[c]) - (E(pc) - E(pn))
        fside = (mc == FLUID) | (mn == FLUID)
        ex_v = np.where(~fside, 0.0, np.where(mc == SOLID, vv[..., c], np.where(inb, shift(vv[..., c], unit(c), 0.0), 0.0)))
        exact = ~fside | (mc == SOLID) | (mn == SOLID)
        out.append(grid_out(u[c], near, exact, ex_v, val))
    return out


def position_change(m, u, p, dt, stray=None):
    """position_change_kernel on the cells within one cell of FLUID: (p_n - p_c) dt, p = 0 off FLUID; 0 on faces with a SOLID side."""
    m = np.asarray(m)
    p = np.asarray(p, dtype=np.float32)
    near = visited(m, stray, 1)
    out = []
    for c in range(3):
        mc, mn, _ = _face_sides(m, c)
        pc = np.where(mc == FLUID, p, 0.0)
        pn = np.where(mn == FLUID, shift(p, unit(c), 0.0), 0.0)
        val = (E(pn) - E(pc)) * float(f32(dt))
        exact = (mc == SOLID) | (mn == SOLID)
        out.append(grid_out(u[c], near, exact, 0.0, val))
    return out


# ------------------------------------------------------------------------------------------------ stages 5 and 12
IN_PLANE = {0: (1, 2), 1: (0, 2), 2: (0, 1)}  # (first, second) in-plane axis of component c, the first fastest


def extrapolate(m, u, mutant=None):
    """extrapolate_kernel: every invalid face with a valid in-plane neighbour takes the average of the valid ones among its 8 in-plane
    neighbours, summed in the shader's order (second axis outer, first axis inner).  mutant = "edges": only the 4 edge neighbours (for the
    tests that show the bounds catch it)."""
    out = []
    for c in range(3):
        val = valid_faces(m, c)
        uc = np.asarray(u[c], dtype=np.float32)
        a, b = IN_PLANE[c]
        avg, num = E(np.zeros(uc.shape)), np.zeros(uc.shape)
        for ob in (-1, 0, 1):
            for oa in (-1, 0, 1):
                if oa == 0 and ob == 0:
                    continue
                if mutant == "edges" and oa != 0 and ob != 0:
                    continue
                d = [0, 0, 0]
                d[a], d[b] = oa, ob
                ok = shift(val, d, False)
                s = avg + E(shift(uc, d, 0.0))
                avg = E(np.where(ok, s.v, avg.v), np.where(ok, s.e, avg.e))
                num += ok
        written = ~val & (num > 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            q = avg / E(np.where(num > 0, num, 1.0))
        out.append(grid_out(uc, written, np.zeros_like(written), 0.0, q))
    return out


# ------------------------------------------------------------------------------------------------ particle stages
CORNERS = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1)]


def clamp_planes(S):
    """1.001f and (float)n - 1.001f per axis (one GPU: the z walls are the grid's)."""
    lo = np.full(3, f32(1.001), dtype=f32)
    hi = np.array([f32(s) - f32(1.001) for s in S], dtype=f32)
    return lo.astype(np.float64), hi.astype(np.float64)


def _cells_of(x, e, S):
    """The cells (trunc, clamped to the grid) the float32 rounding of x +- e can fall into: [n, 3] low and high."""
    lo = np.clip(np.trunc(x.v - e), 0, S - 1).astype(np.int64)
    hi = np.clip(np.trunc(x.v + e), 0, S - 1).astype(np.int64)
    return lo, hi


def _floor_cells(xv, e, S):
    lo = np.clip(np.floor(xv - e), 0, S - 1).astype(np.int64)
    hi = np.clip(np.floor(xv + e), 0, S - 1).astype(np.int64)
    return lo, hi


def _any_in_box(vol, lo, hi):
    """For every particle: (any, all) of the boolean volume vol [z, y, x] over the cell box [lo, hi] (boxes at most 2 wide per axis)."""
    anyv = np.zeros(lo.shape[0], dtype=bool)
    allv = np.ones(lo.shape[0], dtype=bool)
    for bx, by, bz in CORNERS:
        x = np.where(bx, hi[:, 0], lo[:, 0])
        y = np.where(by, hi[:, 1], lo[:, 1])
        z = np.where(bz, hi[:, 2], lo[:, 2])
        v = vol[z, y, x]
        anyv |= v
        allv &= v
    return anyv, allv


def _wall_outcomes(x1, lo, hi):
    """Whether the clamp test (x < lo or x > hi on some axis) can come out true / false within the bound of x1."""
    v, e = x1.v, x1.e
    can_t = ((v - e < lo) | (v + e > hi)).any(axis=1)
    can_f = ((v + e >= lo) & (v - e <= hi)).all(axis=1)
    is_t = ((v < lo) | (v > hi)).any(axis=1)
    return is_t, can_t, can_f


def _cat(xs):
    return E(np.stack([x.v for x in xs], axis=-1), np.stack([x.e for x in xs], axis=-1))


def _hit_branch(x0, mv, dirpos_force):
    """len, dir, maxstep of the hit branch (advect_particles.comp:134-152, density_projection_correct_particles.comp:50-67).  x0 float32
    [n, 3]; mv an E [n, 3]; dirpos_force [n, 3] of -1 (natural), 0 or 1.  Returns (len, dir, maxstep, the natural sign decision, whether
    the sign can go either way)."""
    ln = sqrt(mv[:, 0] * mv[:, 0] + mv[:, 1] * mv[:, 1] + mv[:, 2] * mv[:, 2]) + float(f32(1e-10))
    d = [mv[:, k] / ln for k in range(3)]
    pc = (x0 - np.floor(x0)).astype(f32).astype(np.float64)  # fractf of a float32 value: exact
    step = ln
    nat = np.zeros(x0.shape, dtype=bool)
    amb = np.zeros(x0.shape, dtype=bool)
    for k in range(3):
        nat[:, k] = d[k].v > 0.0
        amb[:, k] = np.abs(mv[:, k].v) <= mv[:, k].e
        pos = np.where(dirpos_force[:, k] < 0, nat[:, k], dirpos_force[:, k] == 1)
        one_minus = 1.0 - E(pc[:, k])
        side = E(np.where(pos, pc[:, k], one_minus.v), np.where(pos, 0.0, one_minus.e))
        ad = E(np.abs(d[k].v), d[k].e)
        with np.errstate(divide="ignore", invalid="ignore"):
            cand = side / ad - float(f32(0.001))
        cand = E(np.where(ad.v > 0.0, cand.v, np.inf), np.where(ad.v > 0.0, cand.e, 0.0))
        step = fmin(step, cand)
    return ln, d, step, nat, amb


def _trilinear_w(w, x, ex):
    """voxel_w_trilinear of the float32 w volume at the float64 point x [n, 3] whose coordinates carry the errors ex [n, 3]."""
    S = np.array([w.shape[2], w.shape[1], w.shape[0]])
    c = x - 0.5
    f = np.floor(c)
    t = c - f
    i0 = f.astype(np.int64)
    lo, hi = np.clip(i0, 0, S - 1), np.clip(i0 + 1, 0, S - 1)
    g = lambda a, b, d: E(w[(hi if d else lo)[:, 2], (hi if b else lo)[:, 1], (hi if a else lo)[:, 0]])
    tx, ty, tz = (E(t[:, k]) for k in range(3))
    c00, c10 = mix(g(0, 0, 0), g(1, 0, 0), tx), mix(g(0, 1, 0), g(1, 1, 0), tx)
    c01, c11 = mix(g(0, 0, 1), g(1, 0, 1), tx), mix(g(0, 1, 1), g(1, 1, 1), tx)
    r = mix(mix(c00, c10, ty), mix(c01, c11, ty), tz)
    spread = float(w.max() - w.min()) if w.size else 0.0
    # the fraction's own error: (x +- 1) and - 0.5 round (u each, relative to the values), plus the position's error
    et = ex + U * (np.abs(x) + np.abs(c))
    return E(r.v, r.e + spread * et.sum(axis=1))


def advect(u, vox, pos, dt, mutant=None):
    """advect_kernel_one (advect_particles.comp:35-194) for the particles pos [n, >= 3] in the face fields u and the fp16 solid volume vox
    (None: no volume).  Returns {"nat": the natural branch, "alt": [(particle indices, branch)], "counts": branch counts}; a branch holds
    "pos" and "rows" (E [n, 3] and three E [n, 4], the rows as stored: (cx, cy, cz, v) per component, B4) and "cells" (low / high cell
    the end point can fall into).  mutant (for the tests that show the bounds catch errors): "b17_fixed" advances component k's
    interpolants by step[axis]; "cy_iy" builds cy with iy in place of iz."""
    u = [np.asarray(a, dtype=np.float32) for a in u]
    S = np.array([u[0].shape[2], u[0].shape[1], u[0].shape[0]])
    p = np.asarray(pos, dtype=f32)[:, :3].copy()
    n = p.shape[0]
    vv = voxel_values(vox, u[0].shape) if vox is not None else None
    dt32 = f32(dt)
    # eaten (:45-64): exact float32 decisions and one float32 addition
    x0 = p.copy()
    eaten = np.zeros(n, dtype=bool)
    axis = np.full(n, -1)
    if vv is not None:
        c = np.clip(np.floor(p).astype(np.int64), 0, S - 1)
        s = vv[c[:, 2], c[:, 1], c[:, 0]]
        eaten = s[:, 3] > 0
        a = np.abs(s[:, :3])
        ax = np.where(a[:, 0] > a[:, 1], np.where(a[:, 0] > a[:, 2], 0, 2), np.where(a[:, 1] > a[:, 2], 1, 2))
        sg = np.sign(s[np.arange(n), ax]).astype(f32)
        i = np.nonzero(eaten)[0]
        x0[i, ax[i]] = (x0[i, ax[i]] + sg[i]).astype(f32)
        axis = np.where(eaten, ax, -1)
    # G2P corners and fractions (:73-92), exact
    corner = np.zeros((3, 8, n))
    fr = np.zeros((3, 3, n))  # fr[axis][component]
    for comp in range(3):
        off = np.full(3, f32(0.5), dtype=f32)
        off[comp] = f32(1.0)
        op = np.maximum(f32(0.0), (x0 - off).astype(f32))
        lo = np.trunc(op).astype(np.int64)
        hi = np.minimum(lo + 1, S - 1)
        lo = np.minimum(lo, S - 1)
        for k, (bx, by, bz) in enumerate(CORNERS):
            corner[comp, k] = u[comp][(hi if bz else lo)[:, 2], (hi if by else lo)[:, 1], (hi if bx else lo)[:, 0]]
        f = (op - np.floor(op)).astype(f32)
        for a_ in range(3):
            fr[a_, comp] = f[:, a_]
    cv = [[E(corner[k, j]) for j in range(8)] for k in range(3)]
    ix, iy, iz = ([E(fr[a_, k]) for k in range(3)] for a_ in range(3))
    nv, cx, cy, cz = [], [], [], []
    for k in range(3):  # :96-112
        v = cv[k]
        vx00, vx01 = mix(v[0], v[1], ix[k]), mix(v[4], v[5], ix[k])
        vx10, vx11 = mix(v[2], v[3], ix[k]), mix(v[6], v[7], ix[k])
        vxy0, vxy1 = mix(vx00, vx10, iy[k]), mix(vx01, vx11, iy[k])
        nv.append(mix(vxy0, vxy1, iz[k]))
        cx.append(mix(mix(v[1], v[3], iy[k]), mix(v[5], v[7], iy[k]), iz[k]) - mix(mix(v[0], v[2], iy[k]), mix(v[4], v[6], iy[k]), iz[k]))
        if mutant == "cy_iy":
            cy.append(mix(vx10, vx11, iy[k]) - mix(vx00, vx01, iy[k]))
        else:
            cy.append(mix(vx10, vx11, iz[k]) - mix(vx00, vx01, iz[k]))
        cz.append(vxy1 - vxy0)

    def trilerp3(a_, b_, c_):
        out = []
        for k in range(3):
            v = cv[k]
            lo_ = mix(mix(v[0], v[1], a_[k]), mix(v[2], v[3], a_[k]), b_[k])
            hi_ = mix(mix(v[4], v[5], a_[k]), mix(v[6], v[7], a_[k]), b_[k])
            out.append(mix(lo_, hi_, c_[k]))
        return out

    def advance(st):
        if mutant == "b17_fixed":  # component k's interpolant along axis a advances by step[a]
            return ([sat(ix[k] + st[0]) for k in range(3)], [sat(iy[k] + st[1]) for k in range(3)], [sat(iz[k] + st[2]) for k in range(3)])
        return ([sat(ix[k] + st[k]) for k in range(3)], [sat(iy[k] + st[k]) for k in range(3)], [sat(iz[k] + st[k]) for k in range(3)])

    half = float(dt32 * f32(0.5))  # exact
    k2 = trilerp3(*advance([nv[k] * half for k in range(3)]))  # RK4 in the cell, :116-126 (B17 as written)
    k3 = trilerp3(*advance([k2[k] * half for k in range(3)]))
    k4 = trilerp3(*advance([k3[k] * float(dt32) for k in range(3)]))
    c6 = E(float(dt32)) * float(f32(1.0 / 6.0))
    mv = _cat([c6 * (nv[k] + 2.0 * (k2[k] + k3[k]) + k4[k]) for k in range(3)])
    x1 = E(x0.astype(np.float64)) + mv
    lo_pl, hi_pl = clamp_planes(S)
    is_wall, can_wall, can_nowall = _wall_outcomes(x1, lo_pl, hi_pl)
    if vv is not None:
        solidv = vv[..., 3] > 0
        nc = np.clip(np.floor(x1.v).astype(np.int64), 0, S - 1)
        is_vox = solidv[nc[:, 2], nc[:, 1], nc[:, 0]]
        a_, l_ = _any_in_box(solidv, *_floor_cells(x1.v, x1.e, S))
        is_hit = is_wall | is_vox
        can_hit, can_miss = can_wall | a_, can_nowall & ~l_
    else:
        is_vox = np.zeros(n, dtype=bool)
        is_hit, can_hit, can_miss = is_wall, can_wall, can_nowall
    ti0 = np.trunc(x0.astype(np.float64))
    is_same = (ti0 == np.trunc(x1.v)).all(axis=1)
    same_lo, same_hi = np.trunc(x1.v - x1.e), np.trunc(x1.v + x1.e)
    can_same = ((same_lo <= ti0) & (ti0 <= same_hi)).all(axis=1)
    can_diff = ((same_lo != ti0) | (same_hi != ti0)).any(axis=1)
    ln, d, step0, dir_nat, dir_amb = _hit_branch(x0.astype(np.float64), mv, np.full((n, 3), -1))
    w = vv[..., 3].astype(np.float64) if vv is not None else None

    def branch(idx, hit, same, dirpos):
        """The outputs of the particles idx with the hit / same-cell / sign decisions given ([m] bool, [m] bool, [m, 3] of -1 / 0 / 1)."""
        m = len(idx)
        x0i = x0[idx].astype(np.float64)
        mvi, x1i = mv[idx], x1[idx]
        nvi = [nv[k][idx] for k in range(3)]
        _, di, st, _, _ = _hit_branch(x0i, mvi, dirpos)
        mvh = [di[k] * st for k in range(3)]
        push = (same & (w is not None)) & hit
        if w is not None and push.any():
            for k in range(3):
                pa, pb = x1i.v.copy(), x1i.v.copy()
                pa[:, k] -= 1.0
                pb[:, k] += 1.0
                pk = _trilinear_w(w, pa, x1i.e) - _trilinear_w(w, pb, x1i.e)
                t = mvh[k] + pk * (E(float(dt32)) * 50.0)
                mvh[k] = E(np.where(push, t.v, mvh[k].v), np.where(push, t.e, mvh[k].e))
        xo, vo = [], []
        for k in range(3):
            xh = clampv(E(x0i[:, k]) + mvh[k], lo_pl[k], hi_pl[k])
            vh = (di[k] * st) / float(dt32)
            xo.append(E(np.where(hit, xh.v, x1i.v[:, k]), np.where(hit, xh.e, x1i.e[:, k])))
            vo.append(E(np.where(hit, vh.v, nvi[k].v), np.where(hit, vh.e, nvi[k].e)))
        xo = _cat(xo)
        rows = [_cat([cx[0][idx], cx[1][idx], cx[2][idx], vo[0]]), _cat([cy[0][idx], cy[1][idx], cy[2][idx], vo[1]]),
                _cat([cz[0][idx], cz[1][idx], cz[2][idx], vo[2]])]
        cl, ch = _cells_of(xo, xo.e, S)
        return {"idx": idx, "pos": xo, "rows": rows, "cells": (cl, ch), "hit": hit, "same": same, "dirpos": dirpos}

    all_idx = np.arange(n)
    nat = branch(all_idx, is_hit, is_same, np.where(dir_nat, 1, 0))
    # particles within their bound of a decision: every combination of the ambiguous decisions
    amb_hit = can_hit & can_miss
    amb_same = can_same & can_diff & (vv is not None)
    amb_dir = dir_amb & (is_hit | amb_hit)[:, None]
    alt = []
    for i in np.nonzero(amb_hit | amb_same | amb_dir.any(axis=1))[0]:
        hs = [True, False] if amb_hit[i] else [bool(is_hit[i])]
        ss = [True, False] if amb_same[i] else [bool(is_same[i])]
        ds = [[1, 0] if amb_dir[i, k] else [int(dir_nat[i, k])] for k in range(3)]
        for h, s_, *dd in itertools.product(hs, ss, *ds):
            if h == is_hit[i] and s_ == is_same[i] and list(dd) == list(np.where(dir_nat[i], 1, 0)):
                continue
            alt.append((i, h, s_, dd))
    alts = None
    if alt:
        idx = np.array([a[0] for a in alt])
        alts = branch(idx, np.array([a[1] for a in alt]), np.array([a[2] for a in alt]), np.array([a[3] for a in alt]))
    push_n = is_hit & is_same & (vv is not None)
    counts = {"eaten_x": int((axis == 0).sum()), "eaten_y": int((axis == 1).sum()), "eaten_z": int((axis == 2).sum()),
              "wall": int(is_wall.sum()), "voxel": int((is_vox & ~is_wall).sum()), "hit": int(is_hit.sum()), "push": int(push_n.sum()),
              "margin": int(len(set(a[0] for a in alt)))}
    return {"nat": nat, "alt": alts, "counts": counts, "n": n, "dims": tuple(S), "w": np.asarray(pos, dtype=f32)[:, 3]}


def correct(u, m, pos, mutant=None):
    """correct_particles_kernel_one (density_projection_correct_particles.comp:25-73) for the displacement fields u and the marker m."""
    u = [np.asarray(a, dtype=np.float32) for a in u]
    m = np.asarray(m)
    S = np.array([u[0].shape[2], u[0].shape[1], u[0].shape[0]])
    x0 = np.asarray(pos, dtype=f32)[:, :3].copy()
    n = x0.shape[0]
    ch = []
    for comp in range(3):
        q = np.maximum(f32(0.0), x0)
        q[:, comp] = np.maximum(f32(0.0), (x0[:, comp] - f32(0.5)).astype(f32))
        c = (q - f32(0.5)).astype(f32)
        fl = np.floor(c)
        t = (c - fl).astype(f32)
        i0 = fl.astype(np.int64)
        lo, hi = np.clip(i0, 0, S - 1), np.clip(i0 + 1, 0, S - 1)
        g = lambda a, b, d: E(u[comp][(hi if d else lo)[:, 2], (hi if b else lo)[:, 1], (hi if a else lo)[:, 0]])
        tx, ty, tz = (E(t[:, k]) for k in range(3))
        c00, c10 = mix(g(0, 0, 0), g(1, 0, 0), tx), mix(g(0, 1, 0), g(1, 1, 0), tx)
        c01, c11 = mix(g(0, 0, 1), g(1, 0, 1), tx), mix(g(0, 1, 1), g(1, 1, 1), tx)
        ch.append(mix(mix(c00, c10, ty), mix(c01, c11, ty), tz))
    chv = _cat(ch)
    x1 = E(x0.astype(np.float64)) + chv
    lo_pl, hi_pl = clamp_planes(S)
    is_wall, can_wall, can_nowall = _wall_outcomes(x1, lo_pl, hi_pl)
    solid = m == SOLID
    nc = np.clip(np.floor(x1.v).astype(np.int64), 0, S - 1)
    is_m = solid[nc[:, 2], nc[:, 1], nc[:, 0]]
    a_, l_ = _any_in_box(solid, *_floor_cells(x1.v, x1.e, S))
    is_hit = is_wall | is_m
    can_hit, can_miss = can_wall | a_, can_nowall & ~l_
    _, _, _, dir_nat, dir_amb = _hit_branch(x0.astype(np.float64), chv, np.full((n, 3), -1))

    def branch(idx, hit, dirpos):
        x0i = x0[idx].astype(np.float64)
        _, di, st, _, _ = _hit_branch(x0i, chv[idx], dirpos)
        x1i = x1[idx]
        xo = []
        for k in range(3):
            xh = clampv(E(x0i[:, k]) + di[k] * st, lo_pl[k], hi_pl[k])
            xo.append(E(np.where(hit, xh.v, x1i.v[:, k]), np.where(hit, xh.e, x1i.e[:, k])))
        return {"idx": idx, "pos": _cat(xo), "hit": hit, "dirpos": dirpos}

    nat = branch(np.arange(n), is_hit, np.where(dir_nat, 1, 0))
    amb_hit = can_hit & can_miss
    amb_dir = dir_amb & (is_hit | amb_hit)[:, None]
    alt = []
    for i in np.nonzero(amb_hit | amb_dir.any(axis=1))[0]:
        hs = [True, False] if amb_hit[i] else [bool(is_hit[i])]
        ds = [[1, 0] if amb_dir[i, k] else [int(dir_nat[i, k])] for k in range(3)]
        for h, *dd in itertools.product(hs, *ds):
            if h == is_hit[i] and list(dd) == list(np.where(dir_nat[i], 1, 0)):
                continue
            alt.append((i, h, dd))
    alts = branch(np.array([a[0] for a in alt]), np.array([a[1] for a in alt]), np.array([a[2] for a in alt])) if alt else None
    counts = {"wall": int(is_wall.sum()), "solid": int((is_m & ~is_wall).sum()), "hit": int(is_hit.sum()), "margin": int(len(set(a[0] for a in alt)))}
    return {"nat": nat, "alt": alts, "counts": counts, "n": n, "dims": tuple(S), "w": np.asarray(pos, dtype=f32)[:, 3]}


def _within(br, got_pos, got_rows):
    """[m] bool: every output of the branch's particles within its bound; and the largest err / bound per particle."""
    idx = br["idx"]
    parts = [(br["pos"], got_pos[idx, :3])]
    if got_rows is not None:
        parts += [(br["rows"][k], got_rows[k][idx]) for k in range(3)]
    ok = np.ones(len(idx), dtype=bool)
    ratio = np.zeros(len(idx))
    for ref, got in parts:
        err = np.abs(np.asarray(got, dtype=np.float64) - ref.v)
        b = bound(ref.e)
        ok &= (err <= b).all(axis=1)
        with np.errstate(invalid="ignore"):
            ratio = np.maximum(ratio, np.nan_to_num((err / b).max(axis=1), nan=np.inf))
    return ok, ratio


def _names(got_rows):
    return ["pos"] + ([f"row{k}" for k in range(3)] if got_rows is not None else [])


def check_particles(got_pos, ref, what, got_rows=None, got_marker=None, keeps_w=True):
    """The kernel's particles (positions [n, 4], rows three [n, 4], the marker after the advection) against advect / correct: every
    particle within the bounds of its natural branch or of one of its alternatives (a margin particle), the fourth position component
    bit for bit (keeps_w), the marker FLUID exactly on the cells of the particles' branches.  Returns (err / bound per particle on the branch taken,
    how many margin particles took an alternative)."""
    got_pos = np.asarray(got_pos, dtype=np.float32)
    n = ref["n"]
    assert got_pos.shape[0] == n, (got_pos.shape, n)
    if keeps_w:  # the kernels carry the fourth component through (the oracle keeps its own bookkeeping there)
        assert np.array_equal(got_pos[:, 3].view(np.uint32), ref["w"].view(np.uint32)), f"{what}: the fourth position component changed"
    ok, ratio = _within(ref["nat"], got_pos, got_rows)
    taken = np.full(n, -1)  # -1: natural branch; else the row of ref["alt"]
    alt = ref["alt"]
    if alt is not None and not ok.all():
        aok, aratio = _within(alt, got_pos, got_rows)
        for j in np.nonzero(aok)[0]:
            i = alt["idx"][j]
            if not ok[i]:
                ok[i], ratio[i], taken[i] = True, aratio[j], j
    if not ok.all():
        i = int(np.nonzero(~ok)[0][0])
        nat = ref["nat"]
        rows = [nat["pos"]] + (nat["rows"] if got_rows is not None else [])
        gots = [got_pos[:, :3]] + (list(got_rows) if got_rows is not None else [])
        worst = None
        for name, r, g in zip(_names(got_rows), rows, gots):
            err = np.abs(np.asarray(g[i], np.float64) - r.v[i])
            b = bound(r.e[i])
            k = int(np.argmax(np.nan_to_num(err - b, nan=np.inf)))
            if not err[k] <= b[k] and worst is None:
                worst = f"{name}[{k}]: kernel {g[i][k]!r}, float64 {r.v[i][k]!r}, bound {b[k]:.3e}"
        nalt = 0 if alt is None else int((alt["idx"] == i).sum())
        raise AssertionError(f"{what}: {int((~ok).sum())} of {n} particles outside the bounds of every branch; first: particle {i}, {worst} "
                             f"(natural branch: hit {bool(nat['hit'][i])}; {nalt} alternative branches)")
    if got_marker is not None:
        got_marker = np.asarray(got_marker)
        cl = ref["nat"]["cells"][0].copy()
        chh = ref["nat"]["cells"][1].copy()
        j = taken >= 0
        if j.any():
            cl[j], chh[j] = alt["cells"][0][taken[j]], alt["cells"][1][taken[j]]
        fl = got_marker == FLUID
        assert ((got_marker == FLUID) | (got_marker == AIR)).all(), f"{what}: the marker holds other values than FLUID and AIR"
        anyf, _ = _any_in_box(fl, cl, chh)
        bad = np.nonzero(~anyf)[0]
        assert bad.size == 0, f"{what}: particle {int(bad[0])} (cells {cl[bad[0]]} .. {chh[bad[0]]}) left no FLUID cell"
        allowed = np.zeros(fl.shape, dtype=bool)
        for bx, by, bz in CORNERS:
            allowed[np.where(bz, chh[:, 2], cl[:, 2]), np.where(by, chh[:, 1], cl[:, 1]), np.where(bx, chh[:, 0], cl[:, 0])] = True
        stray = fl & ~allowed
        assert not stray.any(), f"{what}: FLUID at [z, y, x] = {tuple(int(v) for v in np.argwhere(stray)[0])} where no particle ends"
    return ratio, int((taken >= 0).sum())
