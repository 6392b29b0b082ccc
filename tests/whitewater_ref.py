"""NumPy restatement of the whitewater pass (whitewater_kernels.cu, DESIGN.md §8 "Whitewater") for the tests.

Every expression is the kernels' in float32 with the same order of operations; the kernels are compiled without FMA contraction and with
IEEE division and square root, so that this agrees with them bit for bit from identical inputs.  Grid volumes are (nz, ny, nx) arrays:
the three MAC velocity components u[c] (face i of component c lies between cell i and its +c neighbour), the marker (int8: 1 FLUID,
-1 AIR, 0 SOLID) and the w channel of the solid volume (float32, or None).
"""
from __future__ import annotations

import numpy as np

from tests.flow_ref import Xoshiro

f32 = np.float32
SPRAY, FOAM, BUBBLE = 0, 1, 2
FLUID, AIR, SOLID = 1, -1, 0
SEED_KEY = np.uint64(0xD1B54A32D192ED03)  # WHITEWATER_SEED_KEY


def mix(a, b, t):
    return a * (f32(1) - t) + b * t


def ramp(v, lo, hi):
    return np.fmin(np.fmax((v - f32(lo)) / (f32(hi) - f32(lo)), f32(0)), f32(1))


def seeds(step_count, cells):
    """The emission seed of each cell: (step << 32 | cell) ^ SEED_KEY."""
    return ((np.uint64(step_count) << np.uint64(32)) | np.asarray(cells, dtype=np.uint64)) ^ SEED_KEY


def sample_u(u, x):
    """Advection's MAC trilinear sample of u at the points x (m, 3)."""
    nz, ny, nx = u[0].shape
    S = (nx, ny, nz)
    x = np.asarray(x, dtype=f32)
    out = np.empty((len(x), 3), dtype=f32)
    for c in range(3):
        op = [np.fmax(f32(0), x[:, k] - f32(1.0 if k == c else 0.5)) for k in range(3)]
        lo = [op[k].astype(np.int64) for k in range(3)]
        hi = [np.minimum(lo[k] + 1, S[k] - 1) for k in range(3)]
        lo = [np.minimum(lo[k], S[k] - 1) for k in range(3)]
        ix, iy, iz = (op[k] - np.floor(op[k]) for k in range(3))
        U = u[c]
        at = lambda a, b, d: U[d, b, a]
        c0, c1, c2, c3 = at(lo[0], lo[1], lo[2]), at(hi[0], lo[1], lo[2]), at(lo[0], hi[1], lo[2]), at(hi[0], hi[1], lo[2])
        c4, c5, c6, c7 = at(lo[0], lo[1], hi[2]), at(hi[0], lo[1], hi[2]), at(lo[0], hi[1], hi[2]), at(hi[0], hi[1], hi[2])
        a = mix(mix(c0, c1, ix), mix(c2, c3, ix), iy)
        b = mix(mix(c4, c5, ix), mix(c6, c7, ix), iy)
        out[:, c] = mix(a, b, iz)
    return out


def _cells(shape, x):
    nz, ny, nx = shape
    return [np.clip(np.floor(x[:, k]).astype(np.int64), 0, d - 1) for k, d in enumerate((nx, ny, nz))]


def fluid_count(marker, cx, cy, cz):
    """FLUID cells among the 27 around (cx, cy, cz); cells outside the grid are not FLUID."""
    pad = np.pad(marker == FLUID, 1, constant_values=False)
    a = np.zeros(len(cx), dtype=np.int64)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                a += pad[cz + dz + 1, cy + dy + 1, cx + dx + 1]
    return a


def classify(marker, x, s):
    cx, cy, cz = _cells(marker.shape, np.asarray(x, dtype=f32))
    a = fluid_count(marker, cx, cy, cz)
    own = marker[cz, cy, cx] == FLUID
    return np.where(a < s["spray_below"], SPRAY, np.where(own & (a >= s["bubble_from"]), BUBBLE, FOAM)).astype(np.uint32)


def update(pos, vel, u, marker, vox_w, dt, gravity, s):
    """Phase 1 on the live particles pos / vel (n, 4): returns (pos, vel) of the survivors in their order and the number removed."""
    dt = f32(dt)
    g = np.asarray(gravity, dtype=f32)
    x, v, life = pos[:, :3].astype(f32).copy(), vel[:, :3].astype(f32).copy(), pos[:, 3].astype(f32).copy()
    kind = classify(marker, x, s)
    us = sample_u(u, x)
    spray, bubble, foam = kind == SPRAY, kind == BUBBLE, kind == FOAM
    v[spray] = v[spray] + dt * g
    v[bubble] = (v[bubble] + dt * -(f32(s["buoyancy"]) * g)) + f32(s["drag"]) * (us[bubble] - v[bubble])
    v[foam] = us[foam]
    life[foam] = life[foam] - dt
    x = x + dt * v
    nz, ny, nx = marker.shape
    hi = np.array([nx - 1, ny - 1, nz - 1], dtype=f32)
    gone = ~(life > f32(0)) | ~np.all((x >= f32(1)) & (x < hi), axis=1)
    ok = np.nonzero(~gone)[0]
    c = [x[ok, k].astype(np.int64) for k in range(3)]
    hit = marker[c[2], c[1], c[0]] == SOLID
    if vox_w is not None:
        hit |= vox_w[c[2], c[1], c[0]] > 0
    gone[ok[hit]] = True
    keep = ~gone
    out_pos = np.concatenate([x, life[:, None]], axis=1)[keep].astype(f32)
    out_vel = np.concatenate([v, kind.view(f32)[:, None]], axis=1)[keep].astype(f32)
    return out_pos, out_vel, int(gone.sum())


def _centre(u, x, y, z):
    """Centre velocity of cells (x, y, z); the face below cell 0 reads 0."""
    out = []
    for c, (a, b, d) in enumerate(((x - 1, y, z), (x, y - 1, z), (x, y, z - 1))):
        lower = np.where((a, b, d)[c] >= 0, u[c][np.maximum(d, 0), np.maximum(b, 0), np.maximum(a, 0)], f32(0))
        out.append(f32(0.5) * (lower.astype(f32) + u[c][z, y, x]))
    return out


def band(marker):
    """Linear indices (ascending) of the surface band: FLUID cells off the border with an AIR cell among their 26 neighbours, with the count
    k and the offset sum n of those AIR neighbours."""
    nz, ny, nx = marker.shape
    z, y, x = np.nonzero(marker == FLUID)
    inner = (x > 0) & (y > 0) & (z > 0) & (x < nx - 1) & (y < ny - 1) & (z < nz - 1)
    x, y, z = x[inner], y[inner], z[inner]
    k = np.zeros(len(x), dtype=np.int64)
    n = np.zeros((len(x), 3), dtype=np.int64)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                air = marker[z + dz, y + dy, x + dx] == AIR
                k += air
                n += air[:, None] * np.array([dx, dy, dz])
    m = k > 0
    lin = (z * ny + y) * nx + x
    order = np.argsort(lin[m], kind="stable")
    return lin[m][order], x[m][order], y[m][order], z[m][order], k[m][order], n[m][order]


def potentials(u, marker, s):
    """(lin, I_ta, I_wc, I_k) of every band cell."""
    lin, x, y, z, k, n = band(marker)
    uc = _centre(u, x, y, z)
    xm, xp = _centre(u, x - 1, y, z), _centre(u, x + 1, y, z)
    ym, yp = _centre(u, x, y - 1, z), _centre(u, x, y + 1, z)
    zm, zp = _centre(u, x, y, z - 1), _centre(u, x, y, z + 1)
    h = f32(0.5)
    wx = (yp[2] - ym[2]) * h - (zp[1] - zm[1]) * h
    wy = (zp[0] - zm[0]) * h - (xp[2] - xm[2]) * h
    wz = (xp[1] - xm[1]) * h - (yp[0] - ym[0]) * h
    curl = np.sqrt((wx * wx + wy * wy) + wz * wz)
    uu = (uc[0] * uc[0] + uc[1] * uc[1]) + uc[2] * uc[2]
    energy = h * uu
    i_ta = ramp(curl, *s["trapped_air_range"])
    nz_ = np.any(n != 0, axis=1)
    nl = np.sqrt((n * n).sum(axis=1).astype(f32))
    nf = n.astype(f32)
    dot = (uc[0] * nf[:, 0] + uc[1] * nf[:, 1]) + uc[2] * nf[:, 2]
    crest = nz_ & (dot >= (f32(0.6) * np.sqrt(uu)) * nl)
    i_wc = np.where(crest, ramp(k.astype(f32), *s["wave_crest_range"]), f32(0)).astype(f32)
    i_k = ramp(energy, *s["energy_range"])
    return lin, i_ta, i_wc, i_k


def emit_counts(u, marker, dt, step_count, s):
    """(lin, count, rng) of every band cell: the particles it emits and its generator after the fraction's draw."""
    lin, i_ta, i_wc, i_k = potentials(u, marker, s)
    m = (f32(dt) * (f32(s["trapped_air_rate"]) * i_ta + f32(s["wave_crest_rate"]) * i_wc)) * i_k
    rng = Xoshiro(seeds(step_count, lin))
    draw = rng.next_f32()
    whole = np.floor(m)
    cap = s["max_per_cell"]
    base = np.where(whole >= f32(cap), cap, np.minimum(whole, f32(cap)).astype(np.int64))
    count = np.minimum(base + (draw < m - whole), cap).astype(np.int64)
    return lin, count, rng


def emit(u, marker, dt, step_count, s, room):
    """Phase 2: the new particles in cell order (at most `room`), the total the band asked for."""
    nz, ny, nx = marker.shape
    lin, count, rng = emit_counts(u, marker, dt, step_count, s)
    cap = s["max_per_cell"]
    draws = np.zeros((len(lin), cap, 4), dtype=f32)
    for j in range(cap):
        for a in range(4):
            draws[:, j, a] = rng.next_f32()
    pos = []
    cx, cy, cz = (lin % nx).astype(f32), (lin // nx % ny).astype(f32), (lin // nx // ny).astype(f32)
    for j in range(cap):
        sel = np.nonzero(count > j)[0]
        p = np.stack([cx[sel] + draws[sel, j, 0], cy[sel] + draws[sel, j, 1], cz[sel] + draws[sel, j, 2],
                      f32(s["lifetime_lo"]) + draws[sel, j, 3] * (f32(s["lifetime_hi"]) - f32(s["lifetime_lo"]))], axis=1)
        pos.append((sel * cap + j, p))
    order = np.concatenate([o for o, _ in pos]) if pos else np.zeros(0, dtype=np.int64)
    allp = np.concatenate([p for _, p in pos]).astype(f32) if pos else np.zeros((0, 4), dtype=f32)
    allp = allp[np.argsort(order, kind="stable")]  # cell order, then slot
    total = int(count.sum())
    allp = allp[:min(total, room)]
    v = sample_u(u, allp[:, :3])
    kind = classify(marker, allp[:, :3], s)
    vel = np.concatenate([v, kind.view(f32)[:, None]], axis=1).astype(f32)
    return allp, vel, total


def whitewater_pass(state, u, marker, vox_w, dt, step_count, gravity, s):
    """The whole pass.  state: {"pos", "vel" (n, 4) float32, "counters": [emitted, removed, refused]}; returns the new state."""
    cap = s["max_num_particles"]
    pos, vel, removed = update(state["pos"], state["vel"], u, marker, vox_w, dt, gravity, s)
    new_pos, new_vel, total = emit(u, marker, dt, step_count, s, cap - len(pos))
    emitted = len(new_pos)
    e, r, x = state["counters"]
    return {"pos": np.concatenate([pos, new_pos]).astype(f32), "vel": np.concatenate([vel, new_vel]).astype(f32),
            "counters": [e + emitted, r + removed, x + total - emitted]}
