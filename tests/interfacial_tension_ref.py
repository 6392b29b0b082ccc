"""NumPy restatement of the interfacial tension rule (surface_tension_kernels.cu, DESIGN.md §8 "Interfacial tension"): int64 for the phase
field psi and its smoothing phi, float64 for the curvature (the free surface's formula, tests/surface_tension_ref.py), float32 for the
ghost values and their face coefficients.  Volumes are [z, y, x]; the border of a marker volume is SOLID.  Face arrays of a density table
follow divergence_remove's layout: beta[c][z, y, x] is the face between the cell and its +c neighbour (c = 0 x, 1 y, 2 z)."""
import numpy as np

from tests import surface_tension_ref as S

SOLID, FLUID, AIR = S.SOLID, S.FLUID, S.AIR
FACES = S.FACES
WALL_COMPENSATION = S.WALL_COMPENSATION
f32 = np.float32
MASK64 = (1 << 64) - 1


def raw_psi(splat_all, splat_b):
    """(2 splat_B - splat_all) >> 8 (int64, 2^-32 units) of the two 2^-40 splats, as hi_B - hi_A - borrow: splat_A = splat_all - splat_B
    modulo 2^64, hi the high 56 bits and borrow = lo_B < lo_A, so that |psi| < 2^56 whatever the splats hold."""
    sall = np.asarray(splat_all, dtype=np.int64).view(np.uint64)
    sb = np.asarray(splat_b, dtype=np.int64).view(np.uint64)
    sa = sall - sb  # modulo 2^64
    hb, ha = (sb >> np.uint64(8)).astype(np.int64), (sa >> np.uint64(8)).astype(np.int64)
    lb, la = sb & np.uint64(255), sa & np.uint64(255)
    return hb - ha - (lb < la).astype(np.int64)


def wall_rule(raw, m):
    """psi (int64): raw + sign(raw) 9 * 2^28 per SOLID face neighbour on non-SOLID cells; on SOLID cells the value of largest magnitude among
    the non-SOLID face neighbours, without one of the edge neighbours, without one of the vertex neighbours (0 without any; of two values of
    equal magnitude the positive one).  Every cell is computed (the kernel writes the cells within 3 of FLUID)."""
    raw = np.asarray(raw, dtype=np.int64)
    nsolid = sum((S.shifted(m, *d, SOLID) == SOLID).astype(np.int64) for d in FACES)
    comp = raw + np.sign(raw) * WALL_COMPENSATION * nsolid
    best = np.zeros_like(comp)
    found = np.zeros(m.shape, dtype=bool)
    for shell in (1, 2, 3):
        sb, sf = np.zeros_like(comp), np.zeros(m.shape, dtype=bool)
        for dz in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dx * dx + dy * dy + dz * dz != shell:
                        continue
                    ok = S.shifted(m, dz, dy, dx, SOLID) != SOLID
                    v = np.where(ok, S.shifted(comp, dz, dy, dx, 0), 0)
                    sb = np.where(better(v, sb), v, sb)
                    sf |= ok
        best = np.where(found, best, sb)
        found |= sf
    return np.where(m == SOLID, best, comp).astype(np.int64)


def better(a, b):
    """a replaces b: larger magnitude, or equal magnitude and larger value."""
    return (np.abs(a) > np.abs(b)) | ((np.abs(a) == np.abs(b)) & (a > b))


def phase_field(splat_all, splat_b, m):
    """phi (int64) of the two splats: the wall rule, then the free surface's 1-2-1 filter."""
    return S.smooth(wall_rule(raw_psi(splat_all, splat_b), m))


def phase_b(phi, m):
    """FLUID cells of phase B (phi > 0)."""
    return (m == FLUID) & (np.asarray(phi) > 0)


def interface_faces(phi, m):
    """[(d, mask)] in the kernels' order +x, +y, +z, -x, -y, -z: FLUID cells whose FLUID face neighbour d has the other phase."""
    b = phase_b(phi, m)
    out = []
    for d in FACES:
        nm, nb = S.shifted(m, *d, SOLID), S.shifted(b, *d, False)
        out.append((d, (m == FLUID) & (nm == FLUID) & (b != nb)))
    return out


def band(phi, m):
    """FLUID cells with an interface face."""
    return np.any([mask for _, mask in interface_faces(phi, m)], axis=0)


def curvature(phi, m):
    """The curvature volume the kernel writes: the free surface's formula on the interface band, clamped to [-2, 2], float32, 0 elsewhere."""
    b = band(phi, m)
    k, _ = S.curvature64(phi, b)
    return np.where(b, np.clip(k, -2.0, 2.0), 0.0).astype(f32)


def interface_field(splat_all, splat_b, m):
    """(phi, kappa): the whole stage-1 measurement."""
    phi = phase_field(splat_all, splat_b, m)
    return phi, curvature(phi, m)


def face_beta(beta, d):
    """The coefficient of each cell's face toward neighbour d (1 without a table)."""
    if beta is None:
        return None
    dz, dy, dx = d
    c = 0 if dx else (1 if dy else 2)
    b = np.asarray(beta[c], dtype=f32)
    return b if dx + dy + dz > 0 else S.shifted(b, dz, dy, dx, f32(0))


def weighted(c, ki, kj, bf):
    """beta_f g_f in float32 (g_f alone without a table)."""
    g = S.ghost(c, ki, kj)
    return g if bf is None else (np.asarray(bf, dtype=f32) * g).astype(f32)


def rhs_after(rhs, m, phi, kappa, dt, s, beta=None):
    """The right-hand side after the stage-1 correction: each band cell adds +beta g (phase B) or -beta g (phase A) over its interface faces
    in the order +x, +y, +z, -x, -y, -z into a float32 sum, then rhs + sum."""
    c = S.ghost_scale(dt, s)
    b = phase_b(phi, m)
    acc = np.zeros(m.shape, dtype=f32)
    anyf = np.zeros(m.shape, dtype=bool)
    for d, mask in interface_faces(phi, m):
        w = weighted(c, kappa, S.shifted(kappa, *d, f32(0)), face_beta(beta, d))
        acc = np.where(mask, np.where(b, acc + w, acc - w).astype(f32), acc)
        anyf |= mask
    rhs = np.asarray(rhs, dtype=f32)
    return np.where(anyf, (rhs + acc).astype(f32), rhs)


def faces_after(u, m, phi, kappa, dt, s, axis, beta=None):
    """A grid velocity component after the stage-4 correction: on an interface face, u + beta g when its - side is phase B, u - beta g when
    its - side is phase A (float32)."""
    c = S.ghost_scale(dt, s)
    d = [(0, 0, 1), (0, 1, 0), (1, 0, 0)][axis]
    mask = dict(interface_faces(phi, m))[d]
    w = weighted(c, kappa, S.shifted(kappa, *d, f32(0)), None if beta is None else beta[axis])
    u = np.asarray(u, dtype=f32)
    b = phase_b(phi, m)
    return np.where(mask, np.where(b, u + w, u - w).astype(f32), u)


def capillary_limit_ns(s_air, s_ab):
    """The capillary step limit of the larger of the two tensions."""
    return S.capillary_limit_ns(max(float(f32(s_air)), float(f32(s_ab))))
