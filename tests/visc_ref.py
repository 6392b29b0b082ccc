"""float64 restatement of the viscosity stage, written from DESIGN.md §8 "Viscous liquids".  Volumes are [z, y, x]; component c lies along
array axis 2 - c.  Face i of component c lies between cell i and cell i + e_c.

    live        (marker[i] == FLUID or marker[i + e_c] == FLUID) and neither SOLID
    neighbours  the faces i +- e_d of the same component, in the order -x, +x, -y, +y, -z, +z:
                  a SOLID side (either cell SOLID, or outside the grid)  -> Dirichlet, g = component c of the solid volume at the SOLID cell
                                                                           (cell j if SOLID, else j + e_c; 0 outside the grid / without a volume)
                  else one of its cells FLUID                            -> live, coupled
                  else                                                   -> free surface, dropped
    system      (1 + k m_f) x_f - k sum_live x_n = w_f + k sum_dirichlet g_n,  w = u* - gravity_dt[c],  result u = x + gravity_dt[c]
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

SOLID, FLUID, AIR = 0, 1, -1
DIRECTIONS = [(0, -1), (0, 1), (1, -1), (1, 1), (2, -1), (2, 1)]  # (d, sign) in the order of the rule
EPS32 = float(np.finfo(np.float32).eps)


def shift(a, d, sign, fill):
    """b[p] = a[p + sign * e_d], `fill` outside the grid."""
    ax = 2 - d
    out = np.full_like(a, fill)
    src, dst = [slice(None)] * 3, [slice(None)] * 3
    src[ax] = slice(1, None) if sign > 0 else slice(0, -1)
    dst[ax] = slice(0, -1) if sign > 0 else slice(1, None)
    out[tuple(dst)] = a[tuple(src)]
    return out


def live_faces(marker, c):
    mn = shift(marker, c, 1, SOLID)
    return ((marker == FLUID) | (mn == FLUID)) & (marker != SOLID) & (mn != SOLID)


def neighbours(marker, c, vox=None):
    """Per direction: (coupled, dirichlet, g) volumes for the face at every position (meaningful on live faces)."""
    vel = np.zeros(marker.shape) if vox is None else np.asarray(vox, dtype=np.float64)[..., c]
    mn, vn = shift(marker, c, 1, SOLID), shift(vel, c, 1, 0.0)
    out = []
    for d, sign in DIRECTIONS:
        ma, mb = shift(marker, d, sign, SOLID), shift(mn, d, sign, SOLID)
        dirichlet = (ma == SOLID) | (mb == SOLID)
        g = np.where(ma == SOLID, shift(vel, d, sign, 0.0), shift(vn, d, sign, 0.0))
        coupled = ~dirichlet & ((ma == FLUID) | (mb == FLUID))
        out.append((coupled, dirichlet, np.where(dirichlet, g, 0.0)))
    return out


class System:
    """The sparse system of one component: A (csr over the live faces in C order), b, the live mask and the index volume."""

    def __init__(self, marker, c, k, u_star, gravity_dt, vox=None):
        marker = np.asarray(marker)
        self.c, self.k, self.gravity_dt = c, float(k), float(gravity_dt)
        self.live = live_faces(marker, c)
        n = int(self.live.sum())
        self.index = np.full(marker.shape, -1, dtype=np.int64)
        self.index[self.live] = np.arange(n)
        rows = self.index[self.live]
        diag = np.ones(n)
        b = np.asarray(u_star, dtype=np.float64)[self.live] - self.gravity_dt
        ri, ci, vals = [rows], [rows], []
        self.num_dirichlet = np.zeros(n, dtype=np.int64)
        self.dirichlet_nonzero = np.zeros(n, dtype=bool)
        for (d, sign), (coupled, dirichlet, g) in zip(DIRECTIONS, neighbours(marker, c, vox)):
            cp, di = coupled[self.live], dirichlet[self.live]
            diag += self.k * (cp | di)
            b += self.k * g[self.live]
            self.num_dirichlet += di
            self.dirichlet_nonzero |= di & (g[self.live] != 0)
            nb = shift(self.index, d, sign, -1)[self.live]
            assert (nb[cp] >= 0).all(), "a coupled neighbour is not live"
            ri.append(rows[cp])
            ci.append(nb[cp])
            vals.append(np.full(int(cp.sum()), -self.k))
        vals.insert(0, diag)
        self.A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(ri), np.concatenate(ci))), shape=(n, n))
        self.b = b
        self.n = n

    def solve(self):
        """x in float64: a direct solve (splu), or above 40000 unknowns -- where the factorisation of a 3-D stencil takes minutes -- float64 CG
        run until its true residual is below 1e-12 of |b| (the matrix is well conditioned: at most 1 + 12 k)."""
        if self.n == 0:
            return np.zeros(0)
        if self.n <= 40000:
            return spl.splu(self.A.tocsc()).solve(self.b)
        x, info = spl.cg(self.A, self.b, rtol=1e-14, atol=0.0, maxiter=20000)
        assert info == 0 and np.abs(self.b - self.A @ x).max() <= 1e-12 * max(np.abs(self.b).max(), 1e-300)
        return x

    def residual(self, u_result):
        """b - A (u - gravity_dt) for the live faces of a result volume."""
        x = np.asarray(u_result, dtype=np.float64)[self.live] - self.gravity_dt
        return self.b - self.A @ x

    def rounding_bound(self, iterations, u_star, u_result, vox=None):
        """First-order float32 gap between the recurrence's residual and the true one.  Every iteration rounds u += alpha s once (a relative
        eps of |u|, seen through A: |A|_inf <= 1 + 12 k) and forms r -= alpha q with q a row of at most 7 products and 7 additions of values
        bounded by |s| (2 x 7 roundings through |A|_inf) plus the product and the subtraction (2 more); alpha |s| is an update of x and so
        bounded by 2 max |x|.  That is at most (1 + 2 (14 + 2)) eps |A|_inf max |x| per iteration; the start adds one more such term for
        r_0 = b - A x_0.  max |x| is bounded by the largest value in play: the input, the result, gravity_dt and the solid velocities."""
        scale = max(np.abs(np.asarray(u_star, dtype=np.float64)[self.live]).max(initial=0.0), np.abs(np.asarray(u_result, dtype=np.float64)[self.live]).max(initial=0.0))
        scale += abs(self.gravity_dt)
        if vox is not None:
            scale = max(scale, float(np.abs(np.asarray(vox, dtype=np.float64)[..., self.c]).max()))
        return 33.0 * EPS32 * (iterations + 1) * (1.0 + 12.0 * self.k) * scale
