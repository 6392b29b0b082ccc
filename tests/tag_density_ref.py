"""Restatement of liquids of different densities (DESIGN.md §8 "Liquids of different densities") in int64, float32 and float64.

Arrays are [z, y, x] like the taps.  Face arrays follow divergence_remove's layout: beta[c][i] is the face between cell i and its +c
neighbour (c = 0 x, 1 y, 2 z).  Markers: SOLID 0, FLUID 1, AIR -1; the outside of the grid is SOLID.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

SOLID, FLUID, AIR = 0, 1, -1
FRAC_BITS = 20
f32 = np.float32
AXES = (2, 1, 0)  # the array axis of face component c


def q_of(rho):
    """rint(rho * 2^20) of a float32 density, as the library stores it."""
    return int(np.rint(np.float64(f32(rho)) * (1 << FRAC_BITS)))


def particle_cells(pos, shape):
    """The cell P2G marks for each particle: the position clamped to [1, dim - 1], truncated, clamped to dim - 1 (flat [z, y, x] index)."""
    nz, ny, nx = shape
    p = np.asarray(pos, dtype=f32)[:, :3]
    hi = np.array([nx - 1, ny - 1, nz - 1], dtype=f32)
    c = np.minimum(np.maximum(p, f32(1.0)), hi)
    ijk = np.minimum(c.astype(np.int64), (hi).astype(np.int64))
    return (ijk[:, 2] * ny + ijk[:, 1]) * nx + ijk[:, 0]


def cell_density(pos, tags, table, marker):
    """rho_i = float32(S / (n 2^20)) in float64 on FLUID cells, 0 elsewhere; S = sum of rint(rho_tag 2^20) (int64), tags not in `table` 1."""
    marker = np.asarray(marker)
    cells = particle_cells(pos, marker.shape)
    q = np.full(len(cells), 1 << FRAC_BITS, dtype=np.int64)
    tags = np.asarray(tags, dtype=np.uint32)
    for tag, rho in table.items():
        q[tags == np.uint32(tag)] = q_of(rho)
    n = marker.size
    S = np.zeros(n, dtype=np.int64)
    np.add.at(S, cells, q)
    cnt = np.bincount(cells, minlength=n).astype(np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = (S.astype(np.float64) / (cnt.astype(np.float64) * float(1 << FRAC_BITS))).astype(f32)
    fl = marker.ravel() == FLUID
    rho = np.where(fl, np.where(cnt > 0, rho, f32(1.0)), f32(0.0)).astype(f32)
    return rho.reshape(marker.shape)


def _shift(a, c, d, fill):
    """a at the cell d steps along face component c (the outside takes `fill`)."""
    ax = AXES[c]
    out = np.full_like(a, fill)
    src = [slice(None)] * 3
    dst = [slice(None)] * 3
    if d > 0:
        src[ax], dst[ax] = slice(1, None), slice(None, -1)
    else:
        src[ax], dst[ax] = slice(None, -1), slice(1, None)
    out[tuple(dst)] = a[tuple(src)]
    return out


def face_beta(ma, ra, mb, rb, dtype=f32):
    """Coefficient of the face between cells a and b (elementwise): 2 / (ra + rb) between FLUID cells, 1 / r of the FLUID side next to AIR,
    0 with a SOLID side or no FLUID side; the quotients in float64, rounded once to `dtype` (float32: what the library stores)."""
    ra64, rb64 = np.asarray(ra, dtype=f32).astype(np.float64), np.asarray(rb, dtype=f32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        both = (2.0 / (ra64 + rb64)).astype(dtype)
        only_a = (1.0 / ra64).astype(dtype)
        only_b = (1.0 / rb64).astype(dtype)
    solid = (ma == SOLID) | (mb == SOLID)
    out = np.where((ma == FLUID) & (mb == FLUID), both, np.where(ma == FLUID, only_a, np.where(mb == FLUID, only_b, dtype(0))))
    return np.where(solid, dtype(0), out).astype(dtype)


def coefficients(marker, rho, dtype=f32):
    """(beta[3], D, inv_d2) as the library forms them in stage 0: D summed in float32 in the order -x, +x, -y, +y, -z, +z on FLUID cells
    (0 elsewhere), inv_d2 = float32(1 / D^2) in float64 (1 where D = 0 and off FLUID).  dtype = np.float64: the same system unrounded (the
    float64 restatement, whose D is exactly the sum of its couplings)."""
    m = np.asarray(marker).astype(np.int64)
    rho = np.asarray(rho, dtype=f32)
    beta = [face_beta(m, rho, _shift(m, c, +1, SOLID), _shift(rho, c, +1, f32(0)), dtype) for c in range(3)]
    d = np.zeros(m.shape, dtype=dtype)
    for c in range(3):
        d = (d + _shift(beta[c], c, -1, dtype(0))).astype(dtype)  # the -c face is the +c face of the lower neighbour
        d = (d + beta[c]).astype(dtype)
    fl = m == FLUID
    D = np.where(fl, d, dtype(0)).astype(dtype)
    with np.errstate(divide="ignore"):
        inv = (1.0 / (D.astype(np.float64) ** 2)).astype(f32)
    inv = np.where(fl & (D != 0), inv, f32(1.0)).astype(f32)
    return beta, D, inv


def apply_w(beta, D, fl, x):
    """(A x) in float64 on FLUID cells, 0 elsewhere; x must be 0 off FLUID."""
    x = np.asarray(x, dtype=np.float64)
    s = np.zeros(x.shape)
    for c in (2, 1, 0):  # pcg_ref.nbr_sum's order
        b = beta[c].astype(np.float64)
        s = s + _shift(b, c, -1, 0.0) * _shift(x, c, -1, 0.0)
        s = s + b * _shift(x, c, +1, 0.0)
    return np.where(fl, D.astype(np.float64) * x - s, 0.0)


def apply_w32(beta, D, fl, x):
    """(A x) in float32 with the kernel's order: ((bx- x- + bx+ x+) + (by- y- + by+ y+)) + (bz- z- + bz+ z+), each product rounded, then
    D x - S (NumPy does not fuse: the emulation's convention, as pcg_ref.emulate32's)."""
    x = np.asarray(x, dtype=f32)
    t = []
    for c in range(3):
        t.append((_shift(beta[c], c, -1, f32(0)) * _shift(x, c, -1, f32(0))).astype(f32) + (beta[c] * _shift(x, c, +1, f32(0))).astype(f32))
    S = ((t[0] + t[1]).astype(f32) + t[2]).astype(f32)
    return np.where(fl, (D * x).astype(f32) - S, f32(0)).astype(f32)


def matrix(beta, D, fl):
    """The weighted operator on the FLUID cells as a scipy CSR matrix, and the FLUID cells' flat indices."""
    idx = np.flatnonzero(fl.ravel())
    pos = -np.ones(fl.size, dtype=np.int64)
    pos[idx] = np.arange(len(idx))
    shape = fl.shape
    strides = (1, shape[2], shape[2] * shape[1])
    rows, cols, vals = [idx * 0 + np.arange(len(idx))], [np.arange(len(idx))], [D.ravel()[idx].astype(np.float64)]
    for c in range(3):
        b = beta[c].ravel().astype(np.float64)
        j = idx + strides[c]
        ok = (j < fl.size)
        ok[ok] &= fl.ravel()[j[ok]]
        # the +c neighbour inside the grid: the unrolled flat index wraps only onto border (SOLID) cells, never onto FLUID ones
        rows += [pos[idx[ok]], pos[j[ok]]]
        cols += [pos[j[ok]], pos[idx[ok]]]
        vals += [-b[idx[ok]], -b[idx[ok]]]
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(len(idx), len(idx)))
    return A, idx


def divergence(u, marker):
    """The stage-1 rhs with solids at rest: sum over the axes of u(+face) - u(-face), a face with a SOLID side carrying 0."""
    m = np.asarray(marker)
    out = np.zeros(m.shape)
    for c in range(3):
        uu = np.where((m == SOLID) | (_shift(m, c, +1, SOLID) == SOLID), 0.0, np.asarray(u[c], dtype=np.float64))
        out += uu - _shift(uu, c, -1, 0.0)
    return np.where(m == FLUID, out, 0.0)


def project64(u, marker, beta, p):
    """u = u* - beta (p_i - p_j) on the faces with a FLUID side and no SOLID side (float64); 0 with a SOLID side."""
    m = np.asarray(marker)
    p = np.where(m == FLUID, np.asarray(p, dtype=np.float64), 0.0)
    out = []
    for c in range(3):
        mn = _shift(m, c, +1, SOLID)
        live = ((m == FLUID) | (mn == FLUID)) & (m != SOLID) & (mn != SOLID)
        v = np.asarray(u[c], dtype=np.float64) - beta[c].astype(np.float64) * (p - _shift(p, c, +1, 0.0))
        out.append(np.where(live, v, 0.0))
    return out


def project32(u, marker, beta, p):
    """Stage 4's live faces in float32: __fsub_rn(u, __fmul_rn(beta, __fsub_rn(p_i, p_j))); the mask of the faces it writes that way."""
    m = np.asarray(marker)
    p = np.where(m == FLUID, np.asarray(p, dtype=f32), f32(0)).astype(f32)
    out, masks = [], []
    for c in range(3):
        mn = _shift(m, c, +1, SOLID)
        live = ((m == FLUID) | (mn == FLUID)) & (m != SOLID) & (mn != SOLID)
        dp = (p - _shift(p, c, +1, f32(0))).astype(f32)
        out.append((np.asarray(u[c], dtype=f32) - (beta[c] * dp).astype(f32)).astype(f32))
        masks.append(live)
    return out, masks


def solve64(A, b):
    """The exact solution of the weighted system (sparse direct, float64)."""
    return spla.spsolve(A.tocsc(), b)


def cg64(beta, D, inv, fl, b, p0, iterations):
    """The solve's recurrence in float64 on the float32 coefficients (z = r * inv_d2): [(p_{k+1}, alpha_k, sigma_k)] for k < iterations,
    with pcg.cu's epsilon guards."""
    eps = 1e-10
    A = lambda x: apply_w(beta, D, fl, x)
    p = np.where(fl, np.asarray(p0, dtype=np.float64), 0.0)
    r = np.where(fl, np.asarray(b, dtype=np.float64), 0.0) - A(p)
    z = np.where(fl, r * inv.astype(np.float64), 0.0)
    sigma, beta_k, s = float(np.sum(z * r)), 0.0, np.zeros(p.shape)
    out = []
    for _ in range(iterations):
        s = z + beta_k * s
        As = A(s)
        den = float(np.sum(s * As))
        alpha = sigma / (den + (-eps if den < 0 else eps))
        p = p + alpha * s
        r = r - alpha * As
        out.append((p.copy(), alpha, sigma))
        z = np.where(fl, r * inv.astype(np.float64), 0.0)
        zr = float(np.sum(z * r))
        beta_k = zr / (sigma + (-eps if sigma < 0 else eps))
        sigma = zr
    return out
