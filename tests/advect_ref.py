"""Float64 NumPy restatement of the DECISIONS of the particle stages that meet solids: advection (advect_particles.comp:35-173, fluid_kernels.cu
advect_kernel_one) and the density correction (density_projection_correct_particles.comp:25-73).  It says which branch every particle has to take
-- eaten by a moving wall and along which axis, hit on a wall clamp or a solid voxel, the same-cell push and whether its smooth sample is clamped at
the grid edge -- and where the unclamped end point x1 lies, so that a test can tell a branch that flipped on round-off (x1 within 1e-5 of a cell
plane or a clamp plane) from a wrong branch.  Volumes are [z, y, x]; positions (x, y, z)."""
import numpy as np

from oracle import oracle as O

f32 = np.float32
CORNERS = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
EDGE = 1e-5


def dims_of(vol):
    return np.array([vol.shape[2], vol.shape[1], vol.shape[0]])


def clamp_planes(S):
    """The clamp planes in float32 arithmetic, as both implementations form them: 1.001f and (float)n - 1.001f."""
    return f32(1.001), np.array([f32(s) - f32(1.001) for s in S], dtype=f32)


def point_index(x, S):
    """SamplerPointClamp: floor, clamped to the grid."""
    return np.clip(np.floor(x).astype(np.int64), 0, S - 1)


def _mix(a, b, t):
    return a * (1.0 - t) + b * t


def _sat(x):
    return np.clip(x, 0.0, 1.0)


def _trilinear_clamp(vol, x):
    """SamplerTrilinearClamp of a scalar volume at texel coordinate x [n, 3]; also says whether a corner index was clamped."""
    S = dims_of(vol)
    c = x - 0.5
    f = np.floor(c)
    t = c - f
    i0 = f.astype(np.int64)
    clamped = ((i0 < 0) | (i0 + 1 > S - 1)).any(axis=1)
    lo, hi = np.clip(i0, 0, S - 1), np.clip(i0 + 1, 0, S - 1)
    g = lambda a, b, d: vol[(hi if d else lo)[:, 2], (hi if b else lo)[:, 1], (hi if a else lo)[:, 0]]
    c00 = _mix(g(0, 0, 0), g(1, 0, 0), t[:, 0])
    c10 = _mix(g(0, 1, 0), g(1, 1, 0), t[:, 0])
    c01 = _mix(g(0, 0, 1), g(1, 0, 1), t[:, 0])
    c11 = _mix(g(0, 1, 1), g(1, 1, 1), t[:, 0])
    return _mix(_mix(c00, c10, t[:, 1]), _mix(c01, c11, t[:, 1]), t[:, 2]), clamped


def near_plane(x1, S):
    """x1 within EDGE of an integer plane (floor / trunc decisions) or of a clamp plane."""
    lo, hi = clamp_planes(S)
    d = np.minimum(np.abs(x1 - np.round(x1)), np.minimum(np.abs(x1 - float(lo)), np.abs(x1 - hi.astype(np.float64))))
    return (d < EDGE).any(axis=1)


def advect(u, vox, pos, dt):
    """Branches of advection for the particles `pos` [n, >= 3] in the face fields u = (ux, uy, uz) and the solid volume vox [nz, ny, nx, 4]
    (the float32 values of the fp16 volume).  Returns a dict of per-particle arrays."""
    S = dims_of(u[0])
    p = np.asarray(pos, dtype=f32)[:, :3]
    n = p.shape[0]
    vox = np.asarray(vox, dtype=f32)
    c = point_index(p, S)
    s = vox[c[:, 2], c[:, 1], c[:, 0]]
    eaten = s[:, 3] > 0
    a = np.abs(s[:, :3])
    axis = np.where(a[:, 0] > a[:, 1], np.where(a[:, 0] > a[:, 2], 0, 2), np.where(a[:, 1] > a[:, 2], 1, 2))
    sign = np.sign(s[np.arange(n), axis]).astype(f32)
    x0 = p.copy()
    idx = np.nonzero(eaten)[0]
    x0[idx, axis[idx]] = (x0[idx, axis[idx]] + sign[idx]).astype(f32)  # one float32 addition in both implementations
    x0d = x0.astype(np.float64)
    corners = np.zeros((n, 8, 3))
    it = np.zeros((3, n, 3))  # it[axis][:, component]
    for comp in range(3):
        o = np.full(3, 0.5)
        o[comp] = 1.0
        op = np.maximum(0.0, x0d - o)
        lo = op.astype(np.int64)
        hi = np.minimum(lo + 1, S - 1)
        lo = np.minimum(lo, S - 1)
        U = np.asarray(u[comp], dtype=np.float64)
        for k, (bx, by, bz) in enumerate(CORNERS):
            corners[:, k, comp] = U[(hi if bz else lo)[:, 2], (hi if by else lo)[:, 1], (hi if bx else lo)[:, 0]]
        fr = op - np.floor(op)
        for ax in range(3):
            it[ax][:, comp] = fr[:, ax]

    def trilerp(ix, iy, iz):
        v = corners
        lo_ = _mix(_mix(v[:, 0], v[:, 1], ix), _mix(v[:, 2], v[:, 3], ix), iy)
        hi_ = _mix(_mix(v[:, 4], v[:, 5], ix), _mix(v[:, 6], v[:, 7], ix), iy)
        return _mix(lo_, hi_, iz)

    ix, iy, iz = it
    nv = trilerp(ix, iy, iz)
    st = dt * 0.5 * nv  # quirk B17: component k's three interpolants all advance by step[k]
    k2 = trilerp(_sat(ix + st), _sat(iy + st), _sat(iz + st))
    st = dt * 0.5 * k2
    k3 = trilerp(_sat(ix + st), _sat(iy + st), _sat(iz + st))
    st = dt * k3
    k4 = trilerp(_sat(ix + st), _sat(iy + st), _sat(iz + st))
    mv = dt / 6.0 * (nv + 2.0 * (k2 + k3) + k4)
    x1 = x0d + mv
    lo_pl, hi_pl = clamp_planes(S)
    wall = ((x1 < float(lo_pl)) | (x1 > hi_pl.astype(np.float64))).any(axis=1)
    c1 = point_index(x1, S)
    voxel = ~wall & (vox[c1[:, 2], c1[:, 1], c1[:, 0], 3] > 0)
    hit = wall | voxel
    same = (x0.astype(np.int64) == x1.astype(np.int64)).all(axis=1)
    push = hit & same
    edge = np.zeros(n, dtype=bool)
    w = vox[..., 3].astype(np.float64)
    for k in range(3):
        for sh in (-1.0, 1.0):
            q = x1.copy()
            q[:, k] += sh
            edge |= _trilinear_clamp(w, q)[1]
    return {"x0": x0, "eaten": eaten, "axis": np.where(eaten, axis, -1), "sign": np.where(eaten, sign, 0), "solid_w": s[:, 3],
            "solid_v": s[:, :3], "mv": mv, "x1": x1, "wall": wall, "voxel": voxel, "hit": hit, "push": push, "edge_push": push & edge,
            "near_plane": near_plane(x1, S)}


def correct(u, marker, pos):
    """Branches of the density correction for displacement fields u and the marker volume."""
    S = dims_of(u[0])
    x0 = np.asarray(pos, dtype=f32)[:, :3].astype(np.float64)
    ch = np.zeros_like(x0)
    for comp in range(3):
        o = np.zeros(3)
        o[comp] = 0.5
        ch[:, comp] = _trilinear_clamp(np.asarray(u[comp], dtype=np.float64), np.maximum(0.0, x0 - o))[0]
    x1 = x0 + ch
    lo_pl, hi_pl = clamp_planes(S)
    wall = ((x1 < float(lo_pl)) | (x1 > hi_pl.astype(np.float64))).any(axis=1)
    c1 = point_index(x1, S)
    solid = ~wall & (np.asarray(marker)[c1[:, 2], c1[:, 1], c1[:, 0]] == O.SOLID)
    return {"x1": x1, "wall": wall, "marker": solid, "hit": wall | solid, "near_plane": near_plane(x1, S)}
