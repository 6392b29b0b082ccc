"""NumPy restatement of the flow prologue (sources and drains, DESIGN.md §8) for the tests.

It applies the rules to host arrays with the same float32 expressions as flow_kernels.cu, so that it agrees with the library bit for bit
from identical inputs, and steps the CPU oracle with the prologue in front of every step (``step_with_flow``).
"""
from __future__ import annotations

import numpy as np

M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def clamp_to_grid(dim, v):
    """add_cube's corner clamp (hybrid_fluid.rs:609-617): saturating f32 -> u32, then [1, dim - 1]."""
    v = float(np.float32(v))
    u = 0 if not v > 0.0 else (0xFFFFFFFF if v >= 4294967040.0 else int(v))
    return max(1, min(dim - 1, u))


def make_flow(dims, sources=(), drains=()):
    """Clamped integer boxes: {"sources": [(lo, hi, velocity float32[3])], "drains": [(lo, hi)]} (hi exclusive)."""
    box = lambda mn, mx: (tuple(clamp_to_grid(dims[k], mn[k]) for k in range(3)), tuple(clamp_to_grid(dims[k], mx[k]) for k in range(3)))
    return {"sources": [box(mn, mx) + (np.asarray(vel, dtype=np.float32),) for mn, mx, vel in sources],
            "drains": [box(mn, mx) for mn, mx in drains]}


def _rotl(x, k):
    return (x << np.uint64(k)) | (x >> np.uint64(64 - k))


class Xoshiro:
    """Xoshiro256++ seeded through SplitMix64, vectorised over an array of seeds (blub_b200/csrc/xoshiro.hpp)."""

    def __init__(self, seeds):
        state = np.asarray(seeds, dtype=np.uint64).copy()
        self.s = []
        with np.errstate(over="ignore"):
            for _ in range(4):
                state = state + np.uint64(0x9E3779B97F4A7C15)
                z = state.copy()
                z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
                z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
                self.s.append(z ^ (z >> np.uint64(31)))

    def next_u64(self):
        s = self.s
        with np.errstate(over="ignore"):
            result = _rotl(s[0] + s[3], 23) + s[0]
        t = s[1] << np.uint64(17)
        s[2] = s[2] ^ s[0]
        s[3] = s[3] ^ s[1]
        s[1] = s[1] ^ s[2]
        s[0] = s[0] ^ s[3]
        s[2] = s[2] ^ t
        s[3] = _rotl(s[3], 45)
        return result

    def next_f32(self):
        return ((self.next_u64() >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def cells_of(pos, dims):
    """The cell the transfer kernels assign: clamp to [0, dim - 1] (fminf / fmaxf semantics), truncate, clamp to dim - 1."""
    out = []
    for k in range(3):
        x = np.fmin(np.fmax(pos[:, k].astype(np.float32), np.float32(0.0)), np.float32(dims[k] - 1))
        out.append(np.minimum(x.astype(np.int64), dims[k] - 1))
    return out


def _in_box(c, lo, hi):
    return (c[0] >= lo[0]) & (c[0] < hi[0]) & (c[1] >= lo[1]) & (c[1] < hi[1]) & (c[2] >= lo[2]) & (c[2] < hi[2])


def prologue(pos, rows, step_count, dims, capacity, flow, solid=None):
    """One flow prologue.  pos: (n, 4) float32, rows: three (n, 4) float32, solid: bool (nz, ny, nx) or None.
    Returns (pos, rows, (emitted, drained, refused))."""
    nx, ny, nz = dims
    pos = np.asarray(pos, dtype=np.float32)
    rows = [np.asarray(r, dtype=np.float32).copy() for r in rows]
    c = cells_of(pos, dims)
    drained = np.zeros(len(pos), dtype=bool)
    for lo, hi in flow["drains"]:
        drained |= _in_box(c, lo, hi)
    in_source = np.full(len(pos), -1)
    for k, (lo, hi, vel) in enumerate(flow["sources"]):
        m = _in_box(c, lo, hi) & (in_source < 0)
        in_source[m] = k
    for k, (lo, hi, vel) in enumerate(flow["sources"]):  # nozzle: C = 0, v_c = velocity
        m = in_source == k
        for a in range(3):
            rows[a][m] = np.array([0, 0, 0, vel[a]], dtype=np.float32)
    keep = ~drained
    pos, rows = pos[keep], [r[keep] for r in rows]
    cx, cy, cz = (v[keep] for v in c)
    lin = (cz * ny + cy) * nx + cx
    counts = np.bincount(lin, minlength=nx * ny * nz)
    new_pos, new_rows = [], [[], [], []]
    total = 0
    room = capacity - len(pos)
    for k, (lo, hi, vel) in enumerate(flow["sources"]):
        z, y, x = np.meshgrid(np.arange(lo[2], hi[2]), np.arange(lo[1], hi[1]), np.arange(lo[0], hi[0]), indexing="ij")
        x, y, z = x.ravel(), y.ravel(), z.ravel()  # x fastest
        cell = (z * ny + y) * nx + x
        cnt = counts[cell]
        border = (x == 0) | (y == 0) | (z == 0) | (x == nx - 1) | (y == ny - 1) | (z == nz - 1)
        is_solid = solid.reshape(-1)[cell] if solid is not None else np.zeros(len(cell), dtype=bool)
        emit = (cnt < 4) & ~is_solid & ~border
        rng = Xoshiro((np.uint64(step_count) << np.uint64(32)) | cell.astype(np.uint64))
        r = np.empty((len(cell), 8, 3), dtype=np.float32)
        for slot in range(8):
            for a in range(3):
                r[:, slot, a] = rng.next_f32()
        cellf = np.stack([x, y, z], axis=1).astype(np.float32)
        for j in np.nonzero(emit)[0]:
            for slot in range(int(cnt[j]), 8):
                total += 1
                if total > room:
                    continue
                strat = np.array([slot % 2, slot // 2 % 2, slot // 4 % 2], dtype=np.float32)
                p = cellf[j] + (strat * np.float32(0.5) + r[j, slot] * np.float32(0.5))
                new_pos.append([p[0], p[1], p[2], 0.0])
                for a in range(3):
                    new_rows[a].append([0.0, 0.0, 0.0, vel[a]])
    emitted = min(total, room)
    if emitted:
        pos = np.concatenate([pos, np.asarray(new_pos, dtype=np.float32)])
        rows = [np.concatenate([rows[a], np.asarray(new_rows[a], dtype=np.float32)]) for a in range(3)]
    return pos, rows, (emitted, int(drained.sum()), total - emitted)


def step_with_flow(oracle, flow, counters, solid=None, dt=None, stages=(0, 14)):
    """Runs the prologue on an OracleFluid's particles, then stages [from, to) of its step (the prologue belongs to stage 0)."""
    from oracle.oracle import ARR_POS, ARR_ROWX, ARR_ROWY, ARR_ROWZ, DT_120HZ
    dt = DT_120HZ if dt is None else dt
    frm, to = stages
    if frm == 0:
        pos = oracle.particles(ARR_POS).copy()
        rows = [oracle.particles(a).copy() for a in (ARR_ROWX, ARR_ROWY, ARR_ROWZ)]
        step = int(oracle.L.orc_step_counter(oracle.h))
        pos, rows, c = prologue(pos, rows, step, (oracle.nx, oracle.ny, oracle.nz), oracle.max_num_particles, flow, solid)
        oracle.set_particles(pos, *rows)
        for k in range(3):
            counters[k] += c[k]
    oracle.step_stages(dt, frm, to)
