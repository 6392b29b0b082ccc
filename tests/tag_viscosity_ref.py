"""Restatement of liquids of different viscosities (DESIGN.md §8 "Liquids of different viscosities") in int64, float32 and float64.

Volumes are [z, y, x] like the taps; component c lies along array axis 2 - c, face i of component c between cell i and cell i + e_c.  The
classification of faces and neighbours (live, Dirichlet, free surface) is tests/visc_ref.py's.

    q_tag       rint(nu_tag / nu_scale * 2^32) in float64, nu_scale = max(table values, fluid nu); tags not in the table: the fluid's nu
    nu_i        float32((nu_scale * S_i) / (n_i * 2^32)) in float64 on FLUID cells (the fluid's nu without a particle), 0 elsewhere
    nu_fn       face f (cells a, b), neighbour n = f +- e_d (cells j, j + e_c):
                  d = c and the cell between them (b for +, a for -) is FLUID: its nu
                  else float32(((nu_a + nu_b) + (nu_j + nu_j+e_c)) / (number of FLUID cells among them)), non-FLUID cells adding 0
    k_fn        float32(nu_fn * dt)
    system      (1 + sum k_fn) x_f - sum_coupled k_fn x_n = w_f + sum_dirichlet k_fn g_n; a live face whose k_fn are all 0 is no unknown
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from tests import visc_ref as V
from tests.tag_density_ref import particle_cells

SOLID, FLUID, AIR = V.SOLID, V.FLUID, V.AIR
f32 = np.float32
TWO32 = float(1 << 32)


def nu_scale(table, fluid_nu):
    return max([float(f32(fluid_nu))] + [float(f32(v)) for v in table.values()])


def q_of(nu, scale):
    return int(np.rint(float(f32(nu)) / scale * TWO32)) if scale > 0 else 0


def cell_viscosity(pos, tags, table, fluid_nu, marker):
    """nu_i (float32 [z, y, x]) from the particles' cells and tags, exact integer sums."""
    marker = np.asarray(marker)
    scale = nu_scale(table, fluid_nu)
    cells = particle_cells(pos, marker.shape)
    q = np.full(len(cells), q_of(fluid_nu, scale), dtype=np.int64)
    tags = np.asarray(tags, dtype=np.uint32)
    for tag, nu in table.items():
        q[tags == np.uint32(tag)] = q_of(nu, scale)
    n = marker.size
    S = np.zeros(n, dtype=np.int64)
    np.add.at(S, cells, q)
    cnt = np.bincount(cells, minlength=n).astype(np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        nu = ((np.float64(f32(scale)) * S.astype(np.float64)) / (cnt.astype(np.float64) * TWO32)).astype(f32)
    fl = marker.ravel() == FLUID
    nu = np.where(fl, np.where(cnt > 0, nu, f32(fluid_nu)), f32(0.0)).astype(f32)
    return nu.reshape(marker.shape)


def pair_nu(marker, nu, c):
    """Per direction of V.DIRECTIONS: nu_fn (float32) of every face of component c and that neighbour; 0 where the neighbour is dropped."""
    marker = np.asarray(marker)
    nuf = np.where(marker == FLUID, np.asarray(nu, dtype=f32), f32(0)).astype(np.float64)
    mn = V.shift(marker, c, 1, SOLID)
    nun = V.shift(nuf, c, 1, 0.0)
    fa, fb = marker == FLUID, mn == FLUID
    nu_ab = nuf + nun
    out = []
    for (d, sign), (coupled, dirichlet, _) in zip(V.DIRECTIONS, V.neighbours(marker, c)):
        ma, mb = V.shift(marker, d, sign, SOLID), V.shift(mn, d, sign, SOLID)
        nja, njb = V.shift(nuf, d, sign, 0.0), V.shift(nun, d, sign, 0.0)
        cnt = fa.astype(np.int64) + fb + (ma == FLUID) + (mb == FLUID)
        with np.errstate(divide="ignore", invalid="ignore"):
            mean = (nu_ab + (nja + njb)) / cnt
        val = mean.astype(f32)
        if d == c:
            middle_fluid, middle = (fb, nun) if sign > 0 else (fa, nuf)
            val = np.where(middle_fluid, middle.astype(f32), val)
        out.append(np.where(coupled | dirichlet, val, f32(0)).astype(f32))
    return out


def pair_k(marker, nu, c, dt):
    return [(p * f32(dt)).astype(f32) for p in pair_nu(marker, nu, c)]


class PairSystem:
    """The sparse system of one component with per-pair coefficients: A (csr over the unknowns in C order), b, the unknown mask, the index
    volume; the interface of visc_ref.System."""

    def __init__(self, marker, c, nu, dt, u_star, gravity_dt, vox=None):
        marker = np.asarray(marker)
        self.c, self.gravity_dt = c, float(gravity_dt)
        ks = [k.astype(np.float64) for k in pair_k(marker, nu, c, dt)]
        self.k = ks
        nbrs = V.neighbours(marker, c, vox)
        self.classified = V.live_faces(marker, c)
        ksum = sum(ks)
        self.live = self.classified & (ksum > 0)
        n = int(self.live.sum())
        self.index = np.full(marker.shape, -1, dtype=np.int64)
        self.index[self.live] = np.arange(n)
        rows = self.index[self.live]
        diag = np.ones(n)
        b = np.asarray(u_star, dtype=np.float64)[self.live] - self.gravity_dt
        ri, ci, vals = [rows], [rows], []
        self.dirichlet_nonzero = np.zeros(n, dtype=bool)
        self.pair_sets_nonempty = True
        for (d, sign), (coupled, dirichlet, g), k in zip(V.DIRECTIONS, nbrs, ks):
            kl, cp, di = k[self.live], coupled[self.live], dirichlet[self.live]
            diag += np.where(cp | di, kl, 0.0)
            b += np.where(di, kl * g[self.live], 0.0)
            self.dirichlet_nonzero |= di & (g[self.live] != 0) & (kl > 0)
            cpk = cp & (kl > 0)
            nb = V.shift(self.index, d, sign, -1)[self.live]
            assert (nb[cpk] >= 0).all(), "a coupled neighbour with k > 0 is not an unknown"
            ri.append(rows[cpk])
            ci.append(nb[cpk])
            vals.append(-kl[cpk])
        vals.insert(0, diag)
        self.A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(ri), np.concatenate(ci))), shape=(n, n))
        self.b = b
        self.n = n
        self.norm = float(np.abs(self.A).sum(axis=1).max()) if n else 1.0

    solve = V.System.solve
    residual = V.System.residual

    def rounding_bound(self, iterations, u_star, u_result, vox=None):
        """visc_ref.System.rounding_bound with |A|_inf = max row sum of |A| in place of 1 + 12 k."""
        scale = max(np.abs(np.asarray(u_star, dtype=np.float64)[self.live]).max(initial=0.0),
                    np.abs(np.asarray(u_result, dtype=np.float64)[self.live]).max(initial=0.0))
        scale += abs(self.gravity_dt)
        if vox is not None:
            scale = max(scale, float(np.abs(np.asarray(vox, dtype=np.float64)[..., self.c]).max()))
        return 33.0 * V.EPS32 * (iterations + 1) * self.norm * scale


def pair_sets_nonempty(marker, c):
    """Every coupled or Dirichlet neighbour of a live face has at least one FLUID cell in its pair set."""
    marker = np.asarray(marker)
    mn = V.shift(marker, c, 1, SOLID)
    live = V.live_faces(marker, c)
    fa, fb = marker == FLUID, mn == FLUID
    for (d, sign), (coupled, dirichlet, _) in zip(V.DIRECTIONS, V.neighbours(marker, c)):
        ma, mb = V.shift(marker, d, sign, SOLID), V.shift(mn, d, sign, SOLID)
        cnt = fa.astype(np.int64) + fb + (ma == FLUID) + (mb == FLUID)
        if d == c:
            cnt = np.where(fb if sign > 0 else fa, 1, cnt)
        if ((cnt == 0) & live & (coupled | dirichlet)).any():
            return False
    return True
