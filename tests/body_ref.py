"""NumPy restatement of the floating bodies (DESIGN.md §8, "Floating bodies"): the cell rule, the composite solid volume, the load sums and the
integrator with its tank clamp, bit for bit as body_kernels.cu computes them.  Every float32 operation is one rounded NumPy float32 operation in
the kernel's order.  Volumes are [z, y, x]; vectors are (x, y, z); quaternions (w, x, y, z).  A body is a dict as HybridFluid.bodies() returns
it."""
import numpy as np

from tests import load_ref

f32 = np.float32
SOLID = load_ref.SOLID
FOUR_PI_OVER_3 = f32(4.0 * np.pi / 3.0)


def body(shape="box", half_extent=(4, 4, 4), relative_density=0.5, centre=(16, 16, 16), rotation=(1, 0, 0, 0), velocity=(0, 0, 0),
         angular_velocity=(0, 0, 0)):
    ext = (half_extent,) * 3 if np.ndim(half_extent) == 0 else half_extent
    return {"shape": shape, "half_extent": tuple(float(f32(v)) for v in ext), "relative_density": float(f32(relative_density)),
            "centre": tuple(float(f32(v)) for v in centre), "rotation": tuple(float(f32(v)) for v in rotation),
            "velocity": tuple(float(f32(v)) for v in velocity), "angular_velocity": tuple(float(f32(v)) for v in angular_velocity)}


def _v(b, key):
    return [f32(v) for v in b[key]]


def dot3(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def rotation(q):
    """R (3 x 3 nested lists of float32, body -> grid) of the quaternion q = (w, x, y, z)."""
    w, x, y, z = [f32(v) for v in q]
    xx, yy, zz, xy, xz, yz = x * x, y * y, z * z, x * y, x * z, y * z
    wx, wy, wz = w * x, w * y, w * z
    one, two = f32(1), f32(2)
    return [[one - two * (yy + zz), two * (xy - wz), two * (xz + wy)],
            [two * (xy + wz), one - two * (xx + zz), two * (yz - wx)],
            [two * (xz - wy), two * (yz + wx), one - two * (xx + yy)]]


def bounding_extents(b, R=None):
    R = rotation(b["rotation"]) if R is None else R
    h = _v(b, "half_extent")
    if b["shape"] == "sphere":
        return [h[0]] * 3
    return [dot3(abs(R[k][0]), abs(R[k][1]), abs(R[k][2]), h[0], h[1], h[2]) for k in range(3)]


def covered(dims, b):
    """(mask [nz, ny, nx], d = cell centre - c as three float32 volumes) of the cells whose centre lies inside the body."""
    nx, ny, nz = dims
    z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    c = _v(b, "centre")
    d = [(x.astype(f32) + f32(0.5)) - c[0], (y.astype(f32) + f32(0.5)) - c[1], (z.astype(f32) + f32(0.5)) - c[2]]
    h = _v(b, "half_extent")
    if b["shape"] == "sphere":
        return dot3(d[0], d[1], d[2], d[0], d[1], d[2]) <= h[0] * h[0], d
    R = rotation(b["rotation"])
    mask = np.ones(x.shape, dtype=bool)
    for j in range(3):
        mask &= np.abs(dot3(R[0][j], R[1][j], R[2][j], d[0], d[1], d[2])) <= h[j]
    return mask, d


def composite(dims, borrowed, bodies):
    """The composite RGBA16F volume [nz, ny, nx, 4]: the borrowed volume (or zeros), then every body in index order."""
    nx, ny, nz = dims
    out = np.zeros((nz, ny, nx, 4), dtype=np.float16) if borrowed is None else np.array(borrowed, dtype=np.float16)
    for b in bodies:
        mask, d = covered(dims, b)
        v, w = _v(b, "velocity"), _v(b, "angular_velocity")
        vel = [v[0] + (w[1] * d[2] - w[2] * d[1]), v[1] + (w[2] * d[0] - w[0] * d[2]), v[2] + (w[0] * d[1] - w[1] * d[0])]
        for k in range(3):
            out[..., k][mask] = vel[k][mask].astype(np.float16)
        out[..., 3][mask] = np.float16(1.0)
    return out


def loads(marker, p_vel, inv_dt, b):
    """One body's sums {"wetted_faces", "force_fx", "torque_fx"}: the probes' face rule on the SOLID cells the body covers, pivot at the centre."""
    marker = np.asarray(marker)
    nz, ny, nx = marker.shape
    mask, _ = covered((nx, ny, nz), b)
    # SOLID cells outside the body become a value that is neither SOLID nor FLUID: they add no faces and are no fluid neighbour
    m = np.where((marker == SOLID) & ~mask, np.int8(2), marker).astype(marker.dtype)
    return load_ref.solid_loads(m, p_vel, inv_dt, (0, 0, 0), (nx, ny, nz), _v(b, "centre"))


def mass_and_inertia(b):
    h = _v(b, "half_extent")
    rho = f32(b["relative_density"])
    if b["shape"] == "sphere":
        r = h[0]
        m = rho * (((FOUR_PI_OVER_3 * r) * r) * r)
        i = (f32(0.4) * m) * (r * r)
        return m, [i, i, i]
    m = rho * (((f32(8) * h[0]) * h[1]) * h[2])
    hh = [v * v for v in h]
    three = f32(3)
    return m, [(m * (hh[1] + hh[2])) / three, (m * (hh[0] + hh[2])) / three, (m * (hh[0] + hh[1])) / three]


def ll2float(v):
    """__ll2float_rn: int64 to float32, rounded to nearest even (exact through float64 below 2^53)."""
    assert abs(int(v)) < 2 ** 53
    return f32(float(int(v)))


def integrate(b, force_fx, torque_fx, dt, gravity, dims):
    """The body after one step of the integrator with the tank clamp, from the record's sums."""
    dt = f32(dt)
    g = [f32(v) for v in gravity]
    F = [ll2float(v) * f32(2.0 ** -16) for v in force_fx]
    tau = [ll2float(v) * f32(2.0 ** -8) for v in torque_fx]
    m, I = mass_and_inertia(b)
    R = rotation(b["rotation"])
    ab = [dot3(R[0][j], R[1][j], R[2][j], tau[0], tau[1], tau[2]) / I[j] for j in range(3)]
    v, w, c, q = _v(b, "velocity"), _v(b, "angular_velocity"), _v(b, "centre"), _v(b, "rotation")
    for k in range(3):
        v[k] = v[k] + dt * (g[k] + F[k] / m)
        w[k] = w[k] + dt * dot3(R[k][0], R[k][1], R[k][2], ab[0], ab[1], ab[2])
        c[k] = c[k] + dt * v[k]
    dq = [-dot3(w[0], w[1], w[2], q[1], q[2], q[3]),
          q[0] * w[0] + (w[1] * q[3] - w[2] * q[2]),
          q[0] * w[1] + (w[2] * q[1] - w[0] * q[3]),
          q[0] * w[2] + (w[0] * q[2] - w[1] * q[1])]
    half_dt = f32(0.5) * dt
    qn = [q[k] + half_dt * dq[k] for k in range(4)]
    norm = np.sqrt(dot3(qn[0], qn[1], qn[2], qn[0], qn[1], qn[2]) + qn[3] * qn[3])
    q = [qn[k] / norm for k in range(4)]
    out = dict(b, centre=c, velocity=v, angular_velocity=w, rotation=q)
    e = bounding_extents(out)
    for k in range(3):
        if c[k] - e[k] < f32(1):
            c[k] = f32(1) + e[k]
            if v[k] < 0:
                v[k] = f32(0)
        top = f32(dims[k] - 1)
        if c[k] + e[k] > top:
            c[k] = top - e[k]
            if v[k] > 0:
                v[k] = f32(0)
    return {key: (tuple(float(x) for x in val) if isinstance(val, list) else val) for key, val in out.items()}


def normalised(q):
    """set_bodies' normalisation (host, float64 norm): the quaternion it stores."""
    q = [float(f32(v)) for v in q]
    n = np.sqrt(sum(v * v for v in q))
    return tuple(float(f32(v / n)) for v in q)
