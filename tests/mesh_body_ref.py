"""NumPy restatement of the triangle-mesh bodies (DESIGN.md §8, "Mesh bodies"): the vertex transform, the crossing-parity solid fill, the
composite volume, the load sums and the integrator with the asymmetric tank clamp, bit for bit as body_kernels.cu computes them.  float32
steps are one rounded NumPy float32 operation each in the kernel's order; float64 steps are NumPy float64 operations (no FMA on either side).
Also the test meshes and a float64 generalised-winding-number inside test.  Volumes are [z, y, x]; vectors (x, y, z)."""
import numpy as np

from tests import body_ref, load_ref

f32 = np.float32
dot3 = body_ref.dot3


# ---- meshes (outward winding unless said otherwise) ------------------------------------------------------------------------------
def box_mesh(lo, hi):
    x0, y0, z0 = lo
    x1, y1, z1 = hi
    v = np.array([[x0, y0, z0], [x1, y0, z0], [x1, y1, z0], [x0, y1, z0], [x0, y0, z1], [x1, y0, z1], [x1, y1, z1], [x0, y1, z1]], dtype=np.float32)
    t = np.array([[0, 3, 2], [0, 2, 1], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [3, 7, 6], [3, 6, 2], [0, 4, 7], [0, 7, 3], [1, 2, 6], [1, 6, 5]],
                 dtype=np.uint32)
    return v, t


def octahedron(r=1.0):
    v = np.array([[r, 0, 0], [-r, 0, 0], [0, r, 0], [0, -r, 0], [0, 0, r], [0, 0, -r]], dtype=np.float32)
    t = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], dtype=np.uint32)
    return v, t


def icosphere(subdivisions=2, r=1.0):
    p = (1 + 5 ** 0.5) / 2
    v = [(-1, p, 0), (1, p, 0), (-1, -p, 0), (1, -p, 0), (0, -1, p), (0, 1, p), (0, -1, -p), (0, 1, -p), (p, 0, -1), (p, 0, 1), (-p, 0, -1), (-p, 0, 1)]
    v = [np.array(a, dtype=np.float64) / np.linalg.norm(a) for a in v]
    t = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2),
         (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(subdivisions):
        cache, nt = {}, []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = v[a] + v[b]
                v.append(m / np.linalg.norm(m))
                cache[key] = len(v) - 1
            return cache[key]
        for a, b, c in t:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nt += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        t = nt
    return (np.array(v) * r).astype(np.float32), np.array(t, dtype=np.uint32)


def torus(R=2.0, r=0.75, n=24, m=12):
    """About the y axis; n segments around the ring, m around the tube."""
    u, w = np.meshgrid(np.arange(n) * 2 * np.pi / n, np.arange(m) * 2 * np.pi / m, indexing="ij")
    v = np.stack([(R + r * np.cos(w)) * np.cos(u), r * np.sin(w), (R + r * np.cos(w)) * np.sin(u)], -1).reshape(-1, 3)
    t = []
    for i in range(n):
        for j in range(m):
            a, b, c, d = i * m + j, ((i + 1) % n) * m + j, ((i + 1) % n) * m + (j + 1) % m, i * m + (j + 1) % m
            t += [(a, d, c), (a, c, b)]
    return v.astype(np.float32), np.array(t, dtype=np.uint32)


def _merge(parts):
    vs, ts, off = [], [], 0
    for v, t in parts:
        vs.append(v)
        ts.append(t + off)
        off += len(v)
    return np.concatenate(vs), np.concatenate(ts).astype(np.uint32)


def voxel_union_mesh(cells):
    """The closed, outward-wound surface of a union of unit cubes (integer (x, y, z) cells): one quad per exposed face."""
    cells = set(map(tuple, cells))
    verts, index, tris = [], {}, []

    def vid(p):
        if p not in index:
            index[p] = len(verts)
            verts.append(p)
        return index[p]
    for (x, y, z) in sorted(cells):
        for axis in range(3):
            for side in (0, 1):
                nb = [x, y, z]
                nb[axis] += 1 if side else -1
                if tuple(nb) in cells:
                    continue
                a, b = (axis + 1) % 3, (axis + 2) % 3
                corner = []
                for da, db in ((0, 0), (1, 0), (1, 1), (0, 1)):
                    p = [x, y, z]
                    p[axis] += side
                    p[a] += da
                    p[b] += db
                    corner.append(vid(tuple(p)))
                q = corner if side else corner[::-1]
                tris += [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
    return np.array(verts, dtype=np.float32), np.array(tris, dtype=np.uint32)


def l_block():
    """An L of unit cubes: 3 x 1 x 1 along x plus 1 x 2 x 1 up at x = 0 (model units; off-centre centroid, non-diagonal tensor)."""
    return voxel_union_mesh([(0, 0, 0), (1, 0, 0), (2, 0, 0), (0, 1, 0), (0, 2, 0)])


def hollow_box(outer, wall):
    """A box of outer side `outer` cells with a cavity open at the top (walls and floor `wall` thick), as a union of unit cubes."""
    cells = [(x, y, z) for x in range(outer) for y in range(outer) for z in range(outer)
             if not (wall <= x < outer - wall and wall <= z < outer - wall and y >= wall)]
    return voxel_union_mesh(cells)


# ---- mass properties (float64 restatement of mesh_body.cpp) ----------------------------------------------------------------------
def mass_properties(pos, tris, scale):
    p = np.asarray(pos, dtype=np.float64) * float(f32(scale))
    mean = p.mean(axis=0)
    p = p - mean
    a, b, c = p[tris[:, 0]], p[tris[:, 1]], p[tris[:, 2]]
    det = np.einsum("ij,ij->i", a, np.cross(b, c))
    s = a + b + c
    V6 = det.sum()
    sign = -1.0 if V6 < 0 else 1.0
    V = sign * V6 / 6
    com = sign * (det[:, None] * s).sum(0) / 24 / V
    C = sign * np.einsum("i,ijk->jk", det, np.einsum("ij,ik->ijk", a, a) + np.einsum("ij,ik->ijk", b, b) + np.einsum("ij,ik->ijk", c, c)
                         + np.einsum("ij,ik->ijk", s, s)) / 120 - V * np.outer(com, com)
    inertia = np.trace(C) * np.eye(3) - C
    return V, (com + mean) / float(f32(scale)), inertia


# ---- the device rules --------------------------------------------------------------------------------------------------------
def grid_vertices(b, vb):
    """c + R v per vertex in float32, each coordinate c_k + dot3(R_k, v)."""
    R = body_ref.rotation(b["rotation"])
    c = [f32(x) for x in b["centre"]]
    v = np.asarray(vb, dtype=np.float32)
    return np.stack([c[k] + dot3(R[k][0], R[k][1], R[k][2], v[:, 0], v[:, 1], v[:, 2]) for k in range(3)], -1)


def box_offset(R, mid):
    return [dot3(R[k][0], R[k][1], R[k][2], f32(mid[0]), f32(mid[1]), f32(mid[2])) for k in range(3)]


def cube_origin(b, mid):
    R = body_ref.rotation(b["rotation"])
    e = body_ref.bounding_extents(dict(b, shape="box"), R)
    off = box_offset(R, mid)
    return [max(0, int(np.floor((f32(b["centre"][k]) + off[k]) - e[k]))) for k in range(3)]


def edge_function(uy, uz, vy, vz, py, pz):
    swap = uy > vy or (uy == vy and uz > vz)
    ay, az, by, bz = (vy, vz, uy, uz) if swap else (uy, uz, vy, vz)
    ay, az, by, bz = float(ay), float(az), float(by), float(bz)
    e = (by - ay) * (pz - az) - (bz - az) * (py - ay)
    return -e if swap else e


def top_left(dy, dz):
    return dz > 0 or (dz == 0 and dy < 0)


def crossings(vg, tris, lo, cube):
    """{(z, y): [first cell index (local, clamped at 0) per crossing]} of the rows of the launch cube, triangle by triangle."""
    out = {}
    for tri in tris:
        v = [vg[i] for i in tri]
        area = edge_function(v[0][1], v[0][2], v[1][1], v[1][2], v[2][1], v[2][2])
        if area == 0.0:
            continue
        s = 1.0 if area > 0 else -1.0
        tl = []
        for c in range(3):
            a, e = (c + 1) % 3, (c + 2) % 3
            dy, dz = v[e][1] - v[a][1], v[e][2] - v[a][2]
            tl.append(top_left(dy, dz) if area > 0 else top_left(-dy, -dz))
        ys = [v[c][1] for c in range(3)]
        zs = [v[c][2] for c in range(3)]
        y0, y1 = max(lo[1], int(np.floor(min(ys) - f32(0.5)))), min(lo[1] + cube - 1, int(np.ceil(max(ys) - f32(0.5))))
        z0, z1 = max(lo[2], int(np.floor(min(zs) - f32(0.5)))), min(lo[2] + cube - 1, int(np.ceil(max(zs) - f32(0.5))))
        for z in range(z0, z1 + 1):
            for y in range(y0, y1 + 1):
                py, pz = y + 0.5, z + 0.5
                w = []
                for c in range(3):
                    a, e = (c + 1) % 3, (c + 2) % 3
                    w.append(edge_function(v[a][1], v[a][2], v[e][1], v[e][2], py, pz))
                    wn = s * w[c]
                    if not (wn > 0 or (wn == 0 and tl[c])):
                        break
                else:
                    num = (w[0] * float(v[0][0]) + w[1] * float(v[1][0])) + w[2] * float(v[2][0])
                    xs = num / ((w[0] + w[1]) + w[2])
                    first = int(np.floor(xs - 0.5)) + 1 - lo[0]
                    if first < cube:
                        out.setdefault((z, y), []).append(max(first, 0))
    return out


def fill(b, mid, vb, tris, cube):
    """(origin, bits [cube, cube, cube] bool over the launch cube): the crossing parity of every cell."""
    lo = cube_origin(b, mid)
    vg = grid_vertices(b, vb)
    bits = np.zeros((cube, cube, cube), dtype=bool)
    for (z, y), firsts in crossings(vg, tris, lo, cube).items():
        flip = np.zeros(cube, dtype=np.uint8)
        for f in firsts:
            flip[f] ^= 1
        bits[z - lo[2], y - lo[1]] = np.bitwise_xor.accumulate(flip).astype(bool)
    return lo, bits


def covered(dims, b, mesh, cube):
    """(mask [nz, ny, nx], d) as body_ref.covered, for a mesh body; mesh = (mid, body-frame vertices, triangles)."""
    nx, ny, nz = dims
    mid, vb, tris = mesh
    lo, bits = fill(b, mid, vb, tris, cube)
    mask = np.zeros((nz, ny, nx), dtype=bool)
    hz, hy, hx = min(nz, lo[2] + cube) - lo[2], min(ny, lo[1] + cube) - lo[1], min(nx, lo[0] + cube) - lo[0]
    mask[lo[2]:lo[2] + hz, lo[1]:lo[1] + hy, lo[0]:lo[0] + hx] = bits[:hz, :hy, :hx]
    _, d = body_ref.covered(dims, dict(b, shape="sphere", half_extent=(0.0, 0.0, 0.0)))
    return mask, d


def body_mask(dims, b, meshes, i, cube):
    if b["shape"] == "mesh":
        return covered(dims, b, meshes[i], cube)
    return body_ref.covered(dims, b)


def composite(dims, borrowed, bodies, meshes, cube):
    """body_ref.composite with mesh bodies: meshes[i] = (mid, vb, tris) for a mesh body, else None."""
    nx, ny, nz = dims
    out = np.zeros((nz, ny, nx, 4), dtype=np.float16) if borrowed is None else np.array(borrowed, dtype=np.float16)
    for i, b in enumerate(bodies):
        mask, d = body_mask(dims, b, meshes, i, cube)
        v, w = [f32(x) for x in b["velocity"]], [f32(x) for x in b["angular_velocity"]]
        vel = [v[0] + (w[1] * d[2] - w[2] * d[1]), v[1] + (w[2] * d[0] - w[0] * d[2]), v[2] + (w[0] * d[1] - w[1] * d[0])]
        for k in range(3):
            out[..., k][mask] = vel[k][mask].astype(np.float16)
        out[..., 3][mask] = np.float16(1.0)
    return out


def loads(marker, p_vel, inv_dt, b, mesh, cube):
    marker = np.asarray(marker)
    nz, ny, nx = marker.shape
    mask, _ = covered((nx, ny, nz), b, mesh, cube)
    m = np.where((marker == load_ref.SOLID) & ~mask, np.int8(2), marker).astype(marker.dtype)
    return load_ref.solid_loads(m, p_vel, inv_dt, (0, 0, 0), (nx, ny, nz), [f32(x) for x in b["centre"]])


def integrate(b, force_fx, torque_fx, dt, gravity, dims, mass, moments, mid):
    """body_ref.integrate for a mesh body: m and I_b as stored, the clamp on the box centred on c + R mid."""
    dt = f32(dt)
    g = [f32(v) for v in gravity]
    F = [body_ref.ll2float(v) * f32(2.0 ** -16) for v in force_fx]
    tau = [body_ref.ll2float(v) * f32(2.0 ** -8) for v in torque_fx]
    m, I = f32(mass), [f32(x) for x in moments]
    R = body_ref.rotation(b["rotation"])
    ab = [dot3(R[0][j], R[1][j], R[2][j], tau[0], tau[1], tau[2]) / I[j] for j in range(3)]
    v, w, c, q = [[f32(x) for x in b[k]] for k in ("velocity", "angular_velocity", "centre", "rotation")]
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
    R = body_ref.rotation(q)
    e = body_ref.bounding_extents(dict(b, shape="box", rotation=q), R)
    off = box_offset(R, mid)
    for k in range(3):
        if (c[k] + off[k]) - e[k] < f32(1):
            c[k] = (f32(1) + e[k]) - off[k]
            if v[k] < 0:
                v[k] = f32(0)
        top = f32(dims[k] - 1)
        if (c[k] + off[k]) + e[k] > top:
            c[k] = (top - e[k]) - off[k]
            if v[k] > 0:
                v[k] = f32(0)
    return dict(b, centre=tuple(float(x) for x in c), velocity=tuple(float(x) for x in v), angular_velocity=tuple(float(x) for x in w),
                rotation=tuple(float(x) for x in q))


def mid_and_half(props):
    """(mid, half extents) of the body-frame bounds in float32, as the library stores them."""
    lo, hi = [f32(x) for x in props["bounds_lo"]], [f32(x) for x in props["bounds_hi"]]
    return [f32(0.5) * (lo[k] + hi[k]) for k in range(3)], [f32(0.5) * (hi[k] - lo[k]) for k in range(3)]


def cube_side(bodies, mids):
    """The launch cube side of a set: the largest body_cube_side, a mesh body's from the farthest corner of its bounds."""
    side = 0
    for b, mid in zip(bodies, mids):
        h = [float(f32(x)) for x in b["half_extent"]]
        if mid is not None:
            r = max(np.sqrt(sum((float(mid[k]) + (h[k] if c >> k & 1 else -h[k])) ** 2 for k in range(3))) for c in range(8))
        else:
            r = h[0] if b["shape"] == "sphere" else np.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
        side = max(side, int(np.ceil(2 * r)) + 2)
    return side


def quat_to_matrix(q):
    w, x, y, z = [float(v) for v in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def winding_number(vg, tris, points):
    """The float64 generalised winding number (van Oosterom & Strackee solid angles / 4 pi) of the mesh at each point [n, 3]."""
    vg = np.asarray(vg, dtype=np.float64)
    out = np.zeros(len(points))
    for tri in tris:
        a, b, c = vg[tri[0]] - points, vg[tri[1]] - points, vg[tri[2]] - points
        la, lb, lc = np.linalg.norm(a, axis=1), np.linalg.norm(b, axis=1), np.linalg.norm(c, axis=1)
        num = np.einsum("ij,ij->i", a, np.cross(b, c))
        den = la * lb * lc + np.einsum("ij,ij->i", a, b) * lc + np.einsum("ij,ij->i", b, c) * la + np.einsum("ij,ij->i", c, a) * lb
        out += 2 * np.arctan2(num, den)
    return out / (4 * np.pi)


def surface_distance(vg, tris, points):
    """A lower bound of each point's distance to the mesh surface: the distance to each triangle's plane, clamped from below by the
    distance to the triangle's bounding box (exact enough to pick points clear of the surface)."""
    vg = np.asarray(vg, dtype=np.float64)
    best = np.full(len(points), np.inf)
    for tri in tris:
        t = vg[tri]
        n = np.cross(t[1] - t[0], t[2] - t[0])
        n /= np.linalg.norm(n)
        plane = np.abs((points - t[0]) @ n)
        lo, hi = t.min(0), t.max(0)
        box = np.linalg.norm(np.maximum(0, np.maximum(lo - points, points - hi)), axis=1)
        best = np.minimum(best, np.maximum(plane, box))
    return best
