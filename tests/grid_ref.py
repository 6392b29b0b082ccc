"""Float64 restatements of the P2G and density sums, face by face and cell by cell, independent of any grouping, tiling or schedule.
NumPy only.

The (face, particle) pairs are those of transfer_position (transfer_kernels.cu): the position clamped to [lo, dim - 1] (lo = 1.0 for P2G,
0.5 for the density), dual cell d = floor(p - off) (off = 1.0 along the face's axis, 0.5 across it; p - off >= 0 after the clamp, so the
kernels' truncation is a floor), faces / cells d + {0, 1}^3 with the hat weights w = prod sat(1 - |q - p|).  Every face a particle reaches
with w > 0 is one of these eight.  For positions that are float32 values, p - off, q - p and 1 - |q - p| are exact in float32 as well
(their operands are multiples of the ulp of p and the results are not larger than p), so the kernels and this module see the same pairs
and the same 1-D weights; only the products and the sums are rounded in the kernels.

The bounds (p2g_bound, rhs_bound) are per face / cell and come from the kernels' arithmetic, with u = 2^-24 (float32 unit roundoff):
  A = sum w * S over the face's contributions, S = |r_x t_x| + |r_y t_y| + |r_z t_z| + |r_w| (the magnitude of the row's terms),
  D = sum w, V = |sum w * value| / D, G = number of contributions, Smax = max S over the face's contributions.
  scatter form (transfer_kernels.cu: p2g_scatter_kernel, density_scatter_kernel):
    w = (wx wy) wz: 2 roundings; value = r . (t, 1): at most 4 (with or without FMA contraction); w * value: 1; the float32 sum of the
    lanes of one warp peer group: at most 31 roundings whatever the order (32 lanes) -> 38 u A on sum w * value, 33 u D on sum w.
    Each peer-group partial is rounded to 2^-36 (values) / 2^-40 (weights) before the exact integer sums: 2^-37 / 2^-41 per contribution
    (G bounds the number of groups).  A group whose weight rounds to 0 (w < 2^-41) is left out with its value: 2^-41 Smax per
    contribution.  The quotient is formed in double and rounded to float (u V), gravity * dt is added in float (u (V + |g dt|)).
  sequential form (the oracle's list walk): the same per-contribution roundings, then a float32 chain of at most G + 8 additions
    -> (G + 14) u A and (G + 10) u D.  The float32 division and the gravity add as above.
  gather form (p2g_gather_kernel): as the sequential form for the Gn contributions of particles whose primal cell holds at most CROWD_T
    (32) particles.  The Gc contributions of a crowded cell come from p2g_crowded_kernel: each rounded to 2^-24 (2^-25 on both sums) and
    added exactly, then one float conversion that enters the chain as one term; at most 27 such cells reach a face
    -> (Gn + 41) u A + 2^-25 Gc and (Gn + 37) u D + 2^-25 Gc.
  Then |N'/D' - N/D| <= (eN + V eD) / (D - eD) for eN, eD the bounds of the two sums.
  Density rhs: eD as for sum w (density_scatter_kernel, on both transfer paths: 33 u D + 2^-41 G; the oracle: (G + 10) u D); then the conversion to float
  (u D), the 0.5625 per SOLID neighbour (6 float additions: 6 u (D + 3.375)), 1 - d / 8 (u max(1, d / 8)), the division by dt (u |rhs|);
  clamp and max(8, d) are 1-Lipschitz.

Windows.  Every function evaluates either the whole grid or one box of cells, box = ((x0, y0, z0), (x1, y1, z1)) in global cells
(x0 <= x < x1, ...): the arrays then cover the box only, in the global frame (walls, border cells and clamp planes stay the grid's own).  A
particle reaches the faces and cells within REACH = 1 cell of its primal cell, so the sums of a box need only the particles whose cells lie
in the box grown by REACH (the `halo` the sums select particles by); the marker passes read the six neighbours, so density_rhs and
written_faces need the marker of the box grown by one cell, and are exact on the cells of that crop that are not on its rim (an edge of the
crop that is not a wall of the grid).  Particles are taken CHUNK at a time, whole grid or box, so that host memory stays bounded at tens of
millions of particles; the chunks are the same in both forms, so a box equals the same box of the whole grid bit for bit.
"""
import numpy as np

SOLID, FLUID, AIR = 0, 1, -1
U = 2.0 ** -24
REACH = 1         # cells between a particle's primal cell and the farthest face / cell centre it reaches
CHUNK = 1 << 21   # particles per pass


def whole(dims):
    return ((0, 0, 0), tuple(int(n) for n in dims))


def grow(box, halo, dims):
    """The box grown by `halo` cells on every side, cut to the grid."""
    return (tuple(max(0, int(a) - halo) for a in box[0]), tuple(min(int(n), int(b) + halo) for b, n in zip(box[1], dims)))


def crop(a, box):
    """The entries of the global [nz, ny, nx] array `a` in box (a view)."""
    (x0, y0, z0), (x1, y1, z1) = box
    return a[z0:z1, y0:y1, x0:x1]


def inner(frame, box):
    """Index of the entries of box in an array that covers frame (box inside frame)."""
    return tuple(slice(int(b0) - int(f0), int(b1) - int(f0)) for b0, b1, f0 in zip(box[0][::-1], box[1][::-1], frame[0][::-1]))


def clamp_positions(pos, dims, lo):
    p = np.asarray(pos, dtype=np.float64)[:, :3]
    return np.minimum(np.maximum(p, lo), np.asarray(dims, dtype=np.float64) - 1.0)


def _chunks(pos, dims, lo, box, halo):
    """Per CHUNK of particles: (the indices taken, their clamped positions, their primal cells): in the whole grid every particle, in a box
    those whose primal cells lie in the box grown by `halo`."""
    hi_cell = np.asarray(dims, dtype=np.int64) - 1
    full = box == whole(dims)
    blo, bhi = np.asarray(box[0], dtype=np.int64) - halo, np.asarray(box[1], dtype=np.int64) + halo
    for a in range(0, len(pos), CHUNK):
        p = clamp_positions(pos[a:a + CHUNK], dims, lo)
        cell = np.minimum(p.astype(np.int64), hi_cell)
        idx = np.arange(a, a + len(p))
        if not full:
            keep = ((cell >= blo) & (cell < bhi)).all(axis=1)
            idx, p, cell = idx[keep], p[keep], cell[keep]
        yield idx, p, cell


def _corners(p, off, box):
    """Per particle: for each of the 8 corners k (bit 0 = x, 1 = y, 2 = z) of the dual cell d = floor(p - off): the linear index in the
    box, t [n, 3], the weight, and whether the corner lies in the box."""
    lo = np.asarray(box[0], dtype=np.int64)
    ex, ey, ez = (np.asarray(box[1], dtype=np.int64) - lo).tolist()
    d = np.floor(p - off).astype(np.int64)
    out = []
    for k in range(8):
        o = np.array([k & 1, (k >> 1) & 1, k >> 2])
        t = (d + o + off) - p
        w1 = np.clip(1.0 - np.abs(t), 0.0, 1.0)
        c = d + o - lo
        inside = (c[:, 0] >= 0) & (c[:, 0] < ex) & (c[:, 1] >= 0) & (c[:, 1] < ey) & (c[:, 2] >= 0) & (c[:, 2] < ez)
        out.append(((c[:, 2] * ey + c[:, 1]) * ex + c[:, 0], t, w1[:, 0] * w1[:, 1] * w1[:, 2], inside))
    return out


def _shape(box):
    return tuple(int(b) - int(a) for a, b in zip(box[0][::-1], box[1][::-1]))


def _sum(idx, vals, n):
    return np.bincount(idx, weights=vals, minlength=n)


def marker(pos, dims, solid=None, box=None):
    """The marker after P2G: a cell is FLUID iff a particle (clamped to [1, dim - 1]) lies in it, then border and solid cells are SOLID.
    In a box, `solid` covers the box."""
    box = whole(dims) if box is None else box
    lo, hi = np.asarray(box[0], dtype=np.int64), np.asarray(box[1], dtype=np.int64)
    m = np.full(_shape(box), AIR, dtype=np.int8)
    for _, _, c in _chunks(pos, dims, 1.0, box, 0):
        c = c - lo
        m[c[:, 2], c[:, 1], c[:, 0]] = FLUID
    for ax in range(3):  # the grid's border planes that lie in the box
        sl = [slice(None)] * 3
        if lo[ax] == 0:
            sl[2 - ax] = 0
            m[tuple(sl)] = SOLID
        if hi[ax] == dims[ax]:
            sl[2 - ax] = -1
            m[tuple(sl)] = SOLID
    if solid is not None:
        m[np.asarray(solid, dtype=bool)] = SOLID
    return m


CROWD_T = 32  # transfer_kernels.cu: a cell with more particles is summed by p2g_crowded_kernel in the gather form


def p2g_sums(pos, rows, dims, box=None, halo=REACH):
    """For every component c: {"num": sum w * value, "den": sum w, "abs": sum w * S, "count": contributions with w > 0, "crowd":
    those of particles in cells with more than CROWD_T particles, "smax": max S over the contributions} float64 [nz, ny, nx] each (the
    box's shape in a box), over the face (x, y, z) of cell (x, y, z) on the +c side."""
    box = whole(dims) if box is None else box
    n = int(np.prod(_shape(box)))
    # particles per primal cell, over every chunk, in the frame of the cells the particles are taken from
    frame = grow(box, halo, dims)
    flo = np.asarray(frame[0], dtype=np.int64)
    fx, fy, _ = (np.asarray(frame[1], dtype=np.int64) - flo).tolist()
    fkey = lambda cell: ((cell[:, 2] - flo[2]) * fy + cell[:, 1] - flo[1]) * fx + cell[:, 0] - flo[0]
    per_cell = np.zeros(int(np.prod(_shape(frame))), dtype=np.int64)
    for _, _, cell in _chunks(pos, dims, 1.0, box, halo):
        per_cell += np.bincount(fkey(cell), minlength=per_cell.size)
    acc = [{k: np.zeros(n) for k in ("num", "den", "abs", "count", "crowd", "smax")} for _ in range(3)]
    for i, p, cell in _chunks(pos, dims, 1.0, box, halo):
        crowded = per_cell[fkey(cell)] > CROWD_T
        for c in range(3):
            r = np.asarray(rows[c][i], dtype=np.float64)
            off = np.full(3, 0.5)
            off[c] = 1.0
            a = acc[c]
            for idx, t, w, inside in _corners(p, off, box):
                v = (r[:, :3] * t).sum(axis=1) + r[:, 3]
                s = np.abs(r[:, :3] * t).sum(axis=1) + np.abs(r[:, 3])
                live = (w > 0.0) & inside
                idx, w, v, s, cr = idx[live], w[live], v[live], s[live], crowded[live]
                a["num"] += _sum(idx, w * v, n)
                a["den"] += _sum(idx, w, n)
                a["abs"] += _sum(idx, w * s, n)
                a["count"] += np.bincount(idx, minlength=n)
                a["crowd"] += np.bincount(idx[cr], minlength=n)
                np.maximum.at(a["smax"], idx, s)
    return [{k: v.reshape(_shape(box)) for k, v in a.items()} for a in acc]


def written_faces(m, c):
    """Faces P2G writes for component c (at least one side FLUID), and among them those with a SOLID side (written 0)."""
    nb = np.full(m.shape, SOLID, dtype=np.int8)
    ax = 2 - c
    src, dst = [slice(None)] * 3, [slice(None)] * 3
    src[ax], dst[ax] = slice(1, None), slice(0, -1)
    nb[tuple(dst)] = m[tuple(src)]
    writes = (m == FLUID) | (nb == FLUID)
    return writes, writes & ((m == SOLID) | (nb == SOLID))


def p2g_velocity(sums, m, gdt):
    """u[c] = num / den + g dt on the faces P2G writes (den = 0: g dt), 0 on those with a SOLID side; NaN on faces it does not write."""
    out = []
    for c in range(3):
        s = sums[c]
        writes, solid = written_faces(m, c)
        with np.errstate(invalid="ignore", divide="ignore"):
            v = np.where(s["den"] > 0.0, s["num"] / s["den"], 0.0) + float(gdt[c])
        out.append(np.where(writes, np.where(solid, 0.0, v), np.nan))
    return out


def p2g_bound(sums, m, gdt, form):
    """Per-face bound on |u_kernel - u_reference| (module docstring); form "scatter", "gather" or "sequential".  0 on SOLID-side faces (both
    exactly 0)."""
    out = []
    for c in range(3):
        s = sums[c]
        A, D, G, Smax = s["abs"], s["den"], s["count"], s["smax"]
        with np.errstate(invalid="ignore", divide="ignore"):
            V = np.where(D > 0.0, np.abs(s["num"]) / D, 0.0)
        if form == "scatter":
            eN = 38 * U * A + G * (2.0 ** -37 + 2.0 ** -41 * Smax)
            eD = 33 * U * D + G * 2.0 ** -41
        elif form == "gather":
            Gc = s["crowd"]
            eN = (G - Gc + 41) * U * A + Gc * 2.0 ** -25
            eD = (G - Gc + 37) * U * D + Gc * 2.0 ** -25
        elif form == "sequential":
            eN = (G + 14) * U * A
            eD = (G + 10) * U * D
        else:
            raise ValueError(form)
        with np.errstate(invalid="ignore", divide="ignore"):
            q = np.where(D > eD, (eN + V * eD) / (D - eD), np.inf)
        q = np.where(D > 0.0, q, eN + eD)  # no contribution: both are exactly g dt (up to what rounds to nothing)
        b = 1.001 * q + 2 * U * (V + abs(float(gdt[c]))) + 1e-30
        _, solid = written_faces(m, c)
        out.append(np.where(solid, 0.0, b))
    return out


def p2g_bound_terms(s, gdt_c, form):
    """The parts p2g_bound adds up for one component (sums s of p2g_sums, g dt of that component), each as it enters the bound, for
    telling which source of error a face's bound is made of: a ratio close to 1 under a dominant rounding term is tight by design."""
    A, D, G, Smax = s["abs"], s["den"], s["count"], s["smax"]
    with np.errstate(invalid="ignore", divide="ignore"):
        V = np.where(D > 0.0, np.abs(s["num"]) / D, 0.0)
    if form == "scatter":
        num = {"float32 products and peer-group sums (38 u A)": 38 * U * A, "2^-36 quantisation (G 2^-37)": G * 2.0 ** -37,
               "groups of weight below 2^-41 (G 2^-41 Smax)": G * 2.0 ** -41 * Smax}
        eD = 33 * U * D + G * 2.0 ** -41
    elif form == "gather":
        Gc = s["crowd"]
        num = {"float32 chain ((Gn + 41) u A)": (G - Gc + 41) * U * A, "crowded-cell fixed point (Gc 2^-25)": Gc * 2.0 ** -25}
        eD = (G - Gc + 37) * U * D + Gc * 2.0 ** -25
    else:
        raise ValueError(form)
    with np.errstate(invalid="ignore", divide="ignore"):
        scale = np.where(D > eD, 1.001 / (D - eD), np.inf)
        out = {k: v * scale for k, v in num.items()}
        out["error of the weight sum (V eD)"] = V * eD * scale
    out["float division and + g dt (2 u (V + |g dt|))"] = 2 * U * (V + abs(float(gdt_c)))
    return out


def density_sums(pos, dims, box=None, halo=REACH):
    """{"den": sum w, "count": contributions} per cell, float64 [nz, ny, nx] (the box's shape in a box), cells d + {0, 1}^3 of
    d = floor(p - 0.5)."""
    box = whole(dims) if box is None else box
    n = int(np.prod(_shape(box)))
    den, count = np.zeros(n), np.zeros(n)
    for _, p, _ in _chunks(pos, dims, 0.5, box, halo):
        for idx, _, w, inside in _corners(p, np.full(3, 0.5), box):
            live = (w > 0.0) & inside
            den += _sum(idx[live], w[live], n)
            count += np.bincount(idx[live], minlength=n)
    return {"den": den.reshape(_shape(box)), "count": count.reshape(_shape(box))}


def _neighbours(m):
    """Marker of the six face neighbours (SOLID outside the grid), [6, nz, ny, nx]."""
    pad = np.pad(m, 1, constant_values=SOLID)
    nz, ny, nx = m.shape
    sl = lambda dz, dy, dx: pad[1 + dz:1 + dz + nz, 1 + dy:1 + dy + ny, 1 + dx:1 + dx + nx]
    return np.stack([sl(0, 0, 1), sl(0, 1, 0), sl(1, 0, 0), sl(0, 0, -1), sl(0, -1, 0), sl(-1, 0, 0)])


def density_rhs(dsum, m, dt):
    """(1 - (d + 0.5625 k) / 8) clamped to +-0.5 and divided by dt on FLUID cells (d = max(8, .) next to AIR), NaN elsewhere."""
    nb = _neighbours(m)
    d = dsum["den"] + 0.5625 * (nb == SOLID).sum(axis=0)
    d = np.where((nb == AIR).any(axis=0), np.maximum(8.0, d), d)
    rhs = np.clip(1.0 - d / 8.0, -0.5, 0.5) / float(dt)
    return np.where(m == FLUID, rhs, np.nan)


def rhs_bound(dsum, m, dt, form):
    """Per-cell bound on |rhs_kernel - rhs_reference| (module docstring); form "scatter" or "sequential"."""
    D, G = dsum["den"], dsum["count"]
    if form == "scatter":
        eD = 33 * U * D + G * 2.0 ** -41
    elif form == "sequential":
        eD = (G + 10) * U * D
    else:
        raise ValueError(form)
    ed = eD + U * D + 6 * U * (D + 3.375)
    e = (ed / 8.0 + U * np.maximum(1.0, (D + 3.375) / 8.0)) / float(dt) + U * 0.5 / float(dt)
    return np.where(m == FLUID, 1.001 * e + 1e-30, np.nan)


def check(got, want, bound, what, mask=None):
    """max over the checked entries of |got - want| / bound <= 1; returns (that ratio, the bounds checked) for reporting."""
    got = np.asarray(got, dtype=np.float64)
    sel = ~np.isnan(want) if mask is None else (mask & ~np.isnan(want))
    err = np.abs(got[sel] - want[sel])
    b = bound[sel]
    bad = err > b
    if bad.any():
        k = np.argmax(np.where(bad, err - b, -np.inf))
        where = np.argwhere(sel)[k]
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(sel.sum())} entries beyond their bound; worst at [z, y, x] = {tuple(where)}: "
                             f"kernel {got[sel][k]!r}, float64 {want[sel][k]!r}, bound {b[k]:.3e}")
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(err > 0.0, err / b, 0.0)
    return (float(ratio.max()) if err.size else 0.0), b
