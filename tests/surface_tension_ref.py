"""NumPy restatement of the surface tension rule (surface_tension_kernels.cu, DESIGN.md §8 "Surface tension"): int64 for the wall rule and
the smoothed field phi, float64 for the curvature in the same operation order as the kernel (compiled without FMA contraction), float32
for the ghost values.  Volumes are [z, y, x]; the border of a marker volume is SOLID."""
import math

import numpy as np

SOLID, FLUID, AIR = 0, 1, -1
WALL_COMPENSATION = 9 << 28  # 0.5625 in units of 2^-32
# the six face neighbours in the kernels' order: +x, +y, +z, -x, -y, -z, as (dz, dy, dx)
FACES = [(0, 0, 1), (0, 1, 0), (1, 0, 0), (0, 0, -1), (0, -1, 0), (-1, 0, 0)]


def shifted(a, dz, dy, dx, fill):
    """b[z, y, x] = a[z + dz, y + dy, x + dx], `fill` outside the volume."""
    pad = np.pad(a, 1, constant_values=fill)
    nz, ny, nx = a.shape
    return pad[1 + dz:1 + dz + nz, 1 + dy:1 + dy + ny, 1 + dx:1 + dx + nx]


def clamped(a, dz, dy, dx):
    """b[z, y, x] = a at (z + dz, y + dy, x + dx) clamped into the volume."""
    return np.pad(a, 1, mode="edge")[1 + dz:1 + dz + a.shape[0], 1 + dy:1 + dy + a.shape[1], 1 + dx:1 + dx + a.shape[2]]


def near_fluid(m, r):
    """Cells within Chebyshev distance r of a FLUID cell."""
    out = m == FLUID
    for _ in range(r):
        grown = out.copy()
        for dz in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    grown |= shifted(out, dz, dy, dx, False)
        out = grown
    return out


def wall_rule(splat, m):
    """psi (int64): (splat >> 8 as unsigned) + 9 * 2^28 per SOLID face neighbour on non-SOLID cells; on SOLID cells the largest value of the
    non-SOLID face neighbours, without one of the edge neighbours, without one of the vertex neighbours, 0 without any.  Every cell is
    computed (the kernel writes the cells within 3 of FLUID)."""
    base = (np.asarray(splat, dtype=np.int64).view(np.uint64) >> np.uint64(8)).astype(np.int64)
    nsolid = sum((shifted(m, *d, SOLID) == SOLID).astype(np.int64) for d in FACES)
    comp = base + WALL_COMPENSATION * nsolid
    best = np.zeros_like(comp)
    found = np.zeros(m.shape, dtype=bool)
    for shell in (1, 2, 3):
        sb, sf = np.zeros_like(comp), np.zeros(m.shape, dtype=bool)
        for dz in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dx * dx + dy * dy + dz * dz != shell:
                        continue
                    ok = shifted(m, dz, dy, dx, SOLID) != SOLID
                    sb = np.maximum(sb, np.where(ok, shifted(comp, dz, dy, dx, 0), 0))
                    sf |= ok
        best = np.where(found, best, sb)
        found |= sf
    return np.where(m == SOLID, best, comp).astype(np.int64)


def smooth(psi):
    """phi (int64): one 1-2-1 filter per axis, coordinates clamped into the volume.  Every cell is computed (the kernel writes the cells
    within 2 of FLUID)."""
    out = np.zeros_like(psi)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                out += (2 - dx * dx) * (2 - dy * dy) * (2 - dz * dz) * clamped(psi, dz, dy, dx)
    return out


def band(m):
    """FLUID cells with an AIR face neighbour and AIR cells with a FLUID face neighbour."""
    nb = [shifted(m, *d, SOLID) for d in FACES]
    fl = (m == FLUID) & np.any([n == AIR for n in nb], axis=0)
    ai = (m == AIR) & np.any([n == FLUID for n in nb], axis=0)
    return fl | ai


def curvature64(phi, mask):
    """kappa in float64 on `mask` (cells off the border), unclamped, with the kernel's operations in its order; NaN elsewhere.  Returns
    (kappa, zero) with zero = the three integer differences of the gradient are 0."""
    phi = np.asarray(phi, dtype=np.int64)
    z, y, x = np.nonzero(mask)
    f = lambda dx, dy, dz: phi[z + dz, y + dy, x + dx]
    c = f(0, 0, 0)
    ix, iy, iz = f(1, 0, 0) - f(-1, 0, 0), f(0, 1, 0) - f(0, -1, 0), f(0, 0, 1) - f(0, 0, -1)
    d = lambda a: a.astype(np.float64)
    gx, gy, gz = 0.5 * d(ix), 0.5 * d(iy), 0.5 * d(iz)
    fxx = d(f(1, 0, 0) - c) - d(c - f(-1, 0, 0))
    fyy = d(f(0, 1, 0) - c) - d(c - f(0, -1, 0))
    fzz = d(f(0, 0, 1) - c) - d(c - f(0, 0, -1))
    fxy = 0.25 * (d(f(1, 1, 0) - f(1, -1, 0)) - d(f(-1, 1, 0) - f(-1, -1, 0)))
    fxz = 0.25 * (d(f(1, 0, 1) - f(1, 0, -1)) - d(f(-1, 0, 1) - f(-1, 0, -1)))
    fyz = 0.25 * (d(f(0, 1, 1) - f(0, 1, -1)) - d(f(0, -1, 1) - f(0, -1, -1)))
    g2 = gx * gx + gy * gy + gz * gz
    lap = fxx + fyy + fzz
    hess = gx * gx * fxx + gy * gy * fyy + gz * gz * fzz + 2.0 * gx * gy * fxy + 2.0 * gx * gz * fxz + 2.0 * gy * gz * fyz
    zero = (ix == 0) & (iy == 0) & (iz == 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        k = -(lap * g2 - hess) / (g2 * np.sqrt(g2))
    k = np.where(zero, 0.0, k)
    out = np.full(phi.shape, np.nan)
    out[z, y, x] = k
    zout = np.zeros(phi.shape, dtype=bool)
    zout[z, y, x] = zero
    return out, zout


def curvature(phi, m):
    """The curvature volume the kernel writes: float32, clamped to [-2, 2] on the band, 0 elsewhere."""
    b = band(m)
    k, _ = curvature64(phi, b)
    return np.where(b, np.clip(k, -2.0, 2.0), 0.0).astype(np.float32)


def surface_field(splat, m):
    """(phi, kappa) of a splat and a marker volume: the whole stage-1 measurement."""
    phi = smooth(wall_rule(splat, m))
    return phi, curvature(phi, m)


def ghost(c, ki, kj):
    """g = c * (0.5 * (ki + kj)) in float32, c = -(dt * s) in float32."""
    f = np.float32
    return (f(c) * (f(0.5) * (np.asarray(ki, dtype=f) + np.asarray(kj, dtype=f)))).astype(f)


def ghost_scale(dt, sigma):
    return -(np.float32(dt) * np.float32(sigma))


def rhs_after(rhs, m, kappa, dt, sigma):
    """The right-hand side after the stage-1 correction (float32, the kernel's order +x, +y, +z, -x, -y, -z)."""
    c = ghost_scale(dt, sigma)
    s = np.zeros(m.shape, dtype=np.float32)
    anyair = np.zeros(m.shape, dtype=bool)
    for d in FACES:
        air = (m == FLUID) & (shifted(m, *d, SOLID) == AIR)
        s = np.where(air, (s + ghost(c, kappa, shifted(kappa, *d, 0.0))).astype(np.float32), s)
        anyair |= air
    rhs = np.asarray(rhs, dtype=np.float32)
    return np.where(anyair, (rhs + s).astype(np.float32), rhs)


def faces_after(u, m, kappa, dt, sigma, axis):
    """A grid velocity component after the stage-4 correction: u + g where the cell is FLUID and its + neighbour along `axis` (0 = x) AIR,
    u - g the other way round (float32)."""
    c = ghost_scale(dt, sigma)
    d = [(0, 0, 1), (0, 1, 0), (1, 0, 0)][axis]
    mn, kn = shifted(m, *d, SOLID), shifted(kappa, *d, 0.0)
    u = np.asarray(u, dtype=np.float32)
    plus = (m == FLUID) & (mn == AIR)
    minus = (m == AIR) & (mn == FLUID)
    out = np.where(plus, (u + ghost(c, kappa, kn)).astype(np.float32), u)
    return np.where(minus, (u - ghost(c, kn, kappa)).astype(np.float32), out)


def capillary_limit_ns(sigma):
    """floor(1e9 sqrt(1 / (4 pi s))) for a float32 s > 0, saturating at 2^64 - 1."""
    d = math.floor(1e9 * math.sqrt(1.0 / (4.0 * math.pi * float(np.float32(sigma)))))
    return min(d, 2 ** 64 - 1)
