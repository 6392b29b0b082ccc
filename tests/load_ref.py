"""NumPy restatement of the solid load probes (DESIGN.md §8, "Solid load probes"): the box clamp and one record computed from a marker
volume and the velocity solve's pressure, bit for bit as load_kernels.cu computes it.  Volumes are [z, y, x]; boxes, pivots and vectors are
(x, y, z)."""
import numpy as np

SOLID, FLUID = 0, 1
FORCE_FRAC, TORQUE_FRAC = 16, 8


def clamp_closed(dim, v):
    """add_cube's corner conversion (saturating f32 -> u32) clamped to [0, dim] instead of [1, dim - 1]."""
    v = float(np.float32(v))
    u = 0 if not v > 0.0 else (0xFFFFFFFF if v >= 4294967040.0 else int(v))
    return min(dim, u)


def probe_cells(dims, mn, mx):
    """(lo, hi) of a probe box, or None when it is empty after clamping."""
    lo = tuple(clamp_closed(dims[k], mn[k]) for k in range(3))
    hi = tuple(clamp_closed(dims[k], mx[k]) for k in range(3))
    return None if any(h <= l for l, h in zip(lo, hi)) else (lo, hi)


def force_fixed(q):
    """rint(q * 2^16) as int64; q * 2^16 is exact in float32 and float64 alike."""
    return np.rint(np.asarray(q, dtype=np.float32).astype(np.float64) * (1 << FORCE_FRAC)).astype(np.int64)


def torque_fixed(r, q):
    """rint(float32(r * q) * 2^8) as int64: one rounded float32 product, then an exact scaling."""
    v = np.asarray(r, dtype=np.float32) * np.asarray(q, dtype=np.float32)
    return np.rint(v.astype(np.float32).astype(np.float64) * (1 << TORQUE_FRAC)).astype(np.int64)


def solid_loads(marker, p_vel, inv_dt, lo, hi, pivot):
    """One record: {"wetted_faces", "force_fx" [3], "torque_fx" [3]} (Python ints) of the box [lo, hi) with `pivot`."""
    marker = np.asarray(marker)
    p_vel = np.asarray(p_vel, dtype=np.float32)
    inv_dt = np.float32(inv_dt)
    pivot = np.asarray(pivot, dtype=np.float32)
    nz, ny, nx = marker.shape
    dims = (nx, ny, nz)
    box = np.zeros(marker.shape, dtype=bool)
    box[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]] = True
    solid = box & (marker == SOLID)
    force = [0, 0, 0]
    torque = [0, 0, 0]
    faces = 0
    for a in range(3):
        ax = 2 - a
        b1, b2 = (a + 1) % 3, (a + 2) % 3
        for d in (-1, 1):
            # neighbour marker / pressure of every cell, AIR beyond the grid
            nb_m = np.full(marker.shape, -1, dtype=marker.dtype)
            nb_p = np.zeros(marker.shape, dtype=np.float32)
            src = [slice(None)] * 3
            dst = [slice(None)] * 3
            if d > 0:
                src[ax], dst[ax] = slice(1, None), slice(0, -1)
            else:
                src[ax], dst[ax] = slice(0, -1), slice(1, None)
            nb_m[tuple(dst)] = marker[tuple(src)]
            nb_p[tuple(dst)] = p_vel[tuple(src)]
            z, y, x = np.nonzero(solid & (nb_m == FLUID))
            if len(x) == 0:
                continue
            c = (x, y, z)
            q = -(nb_p[z, y, x] * inv_dt)  # float32; the solver's volume holds -p dt / density
            r = []
            for k in range(3):
                if k == a:
                    centre = (c[k] + (1 if d > 0 else 0)).astype(np.float32)
                else:
                    centre = c[k].astype(np.float32) + np.float32(0.5)
                r.append(centre - pivot[k])  # float32
            fq, t1, t2 = force_fixed(q), torque_fixed(r[b2], q), torque_fixed(r[b1], q)
            force[a] += -d * int(fq.sum())
            torque[b1] += -d * int(t1.sum())
            torque[b2] += d * int(t2.sum())
            faces += len(x)
    assert all(dims[k] >= hi[k] for k in range(3))
    return {"wetted_faces": faces, "force_fx": force, "torque_fx": torque}
