"""GPU: the head phases of the P2G and density scatters (transfer_kernels.cu) on particle sets a dam break never makes -- chunks spread so
wide that their tile windows are cut and heads straddle every window face and corner, all 32 lanes of a warp in one cell (several heads per
dual cell), huge and negative velocities, weights that round to 0 -- against an exact integer restatement of the peer groups: the float32
tree of matched_group_sum in the kernel's lane order, rounded as __float2ll_rn does, summed modulo 2^64.  The density accumulator is
compared word for word, the P2G velocities bit for bit through the normalisation's double division."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIMS = (96, 40, 40)  # nx, ny, nz
DT = 1.0 / 120.0


def particles(seed=3):
    """Warps of several kinds, one kind per warp; rows carry only the constant term (r.x = r.y = r.z = 0), so that the value of every face is
    r.w exactly, however the kernel contracts its multiply-adds."""
    rng = np.random.default_rng(seed)
    nx, ny, nz = DIMS
    warps = []
    for w in range(384):
        kind = w % 6
        if kind == 0:  # spread over the whole box: windows cut in z and y, heads straddle their faces
            p = rng.uniform(2.0, [nx - 2.0, ny - 2.0, nz - 2.0], (32, 3))
        elif kind == 1:  # one x row across the grid: windows cut in x
            y, z = rng.uniform(4.0, 30.0, 2)
            p = np.stack([rng.uniform(2.0, nx - 2.0, 32), np.full(32, y), np.full(32, z)], 1)
        elif kind == 2:  # all 32 lanes in one cell: 8 heads per dual cell
            c = rng.integers(3, [nx - 4, ny - 4, nz - 4])
            p = c + rng.uniform(0.0, 1.0, (32, 3))
        elif kind == 3:  # 2 x 2 x 2 cells, 4 particles each
            c = rng.integers(3, [nx - 5, ny - 5, nz - 5])
            p = c + rng.uniform(0.0, 2.0, (32, 3))
        elif kind == 4:  # at cell centres and faces, and a hair off them: weights exactly 0 and weights that round to 0
            c = rng.integers(3, [nx - 4, ny - 4, nz - 4]).astype(np.float32)
            off = rng.choice(np.array([0.0, 0.5, 2e-6, 0.5 + 2e-6, 1.0 - 2e-6, 0.5 - 2e-6], np.float32), (32, 3))
            p = c + off
        else:  # a compact cluster of a few cells
            c = rng.uniform(4.0, [nx - 8, ny - 8, nz - 8])
            p = c + rng.uniform(0.0, 3.0, (32, 3))
        warps.append(p)
    pos = np.zeros((32 * len(warps), 4), np.float32)
    pos[:, :3] = np.concatenate(warps).astype(np.float32)
    n = pos.shape[0]
    rows = [np.zeros((n, 4), np.float32) for _ in range(3)]
    for c in range(3):
        mag = 10.0 ** rng.uniform(-3, 9.7, n)  # up to 5e9: w * value * 2^36 beyond the int64 range for the largest (saturates)
        rows[c][:, 3] = (mag * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    return pos, rows


def f2ll_rn(x):
    """__float2ll_rn of float32 values: round half to even, saturating (NaN -> INT64_MIN)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    out = np.zeros(x.shape, np.int64)
    big = x >= 2.0 ** 63
    small = (x < -(2.0 ** 63)) | np.isnan(x)
    ok = ~(big | small)
    out[ok] = np.rint(x[ok]).astype(np.int64)
    out[big] = np.iinfo(np.int64).max
    out[small] = np.iinfo(np.int64).min
    return out


def group_sums(keys, vals):
    """matched_group_sum over one warp: per key its lanes in ascending order, cut into groups of four by rank, (v0 + v1) + (v2 + v3) in
    float32, at the group's lowest lane.  Returns the head lanes and their sums."""
    heads, sums = [], []
    for key in np.unique(keys):
        lanes = np.nonzero(keys == key)[0]
        for r in range(0, len(lanes), 4):
            g = [vals[l] for l in lanes[r:r + 4]]
            a = g[0] + g[1] if len(g) > 1 else g[0]
            if len(g) > 2:
                a = a + (g[2] + g[3] if len(g) > 3 else g[2])
            heads.append(lanes[r])
            sums.append(a)
    return heads, sums


def sat(x):
    return np.clip(x, np.float32(0.0), np.float32(1.0)).astype(np.float32)


def axis_weights(p, q):
    one = np.float32(1.0)
    return sat(one - np.abs(q - p)), sat(one - np.abs((q + one) - p))


def density_reference(pos):
    nx, ny, nz = DIMS
    lim = np.array([nx - 1.0, ny - 1.0, nz - 1.0], np.float32)
    p = np.minimum(np.maximum(pos[:, :3], np.float32(0.5)), lim).astype(np.float32)
    d = (p - np.float32(0.5)).astype(np.int64)
    q = d.astype(np.float32) + np.float32(0.5)
    w = [axis_weights(p[:, a], q[:, a]) for a in range(3)]
    acc = np.zeros((p.shape[0], 8), np.float32)
    for k in range(8):
        acc[:, k] = w[0][k & 1][:] * w[1][(k >> 1) & 1] * w[2][k >> 2]
    keys = (d[:, 2] * ny + d[:, 1]) * nx + d[:, 0]
    out = np.zeros(nx * ny * nz, np.uint64)
    for b in range(0, p.shape[0], 32):  # positive weights: no sum reaches 2^63
        heads, sums = group_sums(keys[b:b + 32], acc[b:b + 32])
        for h, s in zip(heads, sums):
            base = keys[b + h]
            for k in range(8):
                if s[k] > 0:
                    qv = f2ll_rn(np.float32(s[k]) * np.float32(2.0 ** 40))
                    out[base + (k & 1) + ((k >> 1) & 1) * nx + (k >> 2) * nx * ny] += np.uint64(int(qv) & 0xFFFFFFFFFFFFFFFF)
    return out.view(np.int64).reshape(nz, ny, nx)


def p2g_reference(pos, rows, c):
    """(sum w * value, sum w) per face of component c as int64 words modulo 2^64."""
    nx, ny, nz = DIMS
    lim = np.array([nx - 1.0, ny - 1.0, nz - 1.0], np.float32)
    p = np.minimum(np.maximum(pos[:, :3], np.float32(1.0)), lim).astype(np.float32)
    o = np.array([1.0 if c == a else 0.5 for a in range(3)], np.float32)
    d = (p - o).astype(np.int64)
    q = (d.astype(np.float32) + o).astype(np.float32)
    w = [axis_weights(p[:, a], q[:, a]) for a in range(3)]
    val = rows[c][:, 3]
    acc = np.zeros((p.shape[0], 16), np.float32)
    for k in range(8):
        wk = (w[0][k & 1] * w[1][(k >> 1) & 1] * w[2][k >> 2]).astype(np.float32)
        acc[:, 2 * k] = np.where(wk > 0, wk * val, np.float32(0.0))
        acc[:, 2 * k + 1] = np.where(wk > 0, wk, np.float32(0.0))
    keys = (d[:, 2] * ny + d[:, 1]) * nx + d[:, 0]
    num = np.zeros(nx * ny * nz, np.uint64)
    den = np.zeros(nx * ny * nz, np.uint64)
    m64 = 0xFFFFFFFFFFFFFFFF
    with np.errstate(over="ignore"):  # the sums wrap modulo 2^64, as the kernel's do
        _p2g_sums(p, keys, acc, num, den, m64)
    return num.view(np.int64).reshape(nz, ny, nx), den.view(np.int64).reshape(nz, ny, nx)


def _p2g_sums(p, keys, acc, num, den, m64):
    nx, ny, nz = DIMS
    for b in range(0, p.shape[0], 32):
        heads, sums = group_sums(keys[b:b + 32], acc[b:b + 32])
        for h, s in zip(heads, sums):
            base = keys[b + h]
            for k in range(8):
                wq = int(f2ll_rn(np.float32(s[2 * k + 1]) * np.float32(2.0 ** 40)))
                if wq > 0:
                    nq = int(f2ll_rn(np.float32(s[2 * k]) * np.float32(2.0 ** 36)))
                    f = base + (k & 1) + ((k >> 1) & 1) * nx + (k >> 2) * nx * ny
                    num[f] += np.uint64(nq & m64)
                    den[f] += np.uint64(wq)


def _fluid(pos, rows):
    import blub_b200

    f = blub_b200.HybridFluid(*DIMS, pos.shape[0])
    f.set_gravity_grid([0.0, 0.0, 0.0])
    f.set_particles(pos, *rows)
    return f


def test_density_scatter_heads_match_the_integer_restatement():
    from blub_b200 import fluid as F

    pos, rows = particles()
    f = _fluid(pos, rows)
    f.step_stages(DT, 9, 10)
    got = f.download_grid(F.TAP_DENSITY)
    want = density_reference(pos)
    assert np.count_nonzero(want) > 10000
    bad = np.nonzero(got != want)
    assert bad[0].size == 0, f"{bad[0].size} cells differ, first at (z, y, x) = {[int(b[0]) for b in bad]}"


def test_p2g_scatter_heads_match_the_integer_restatement():
    from blub_b200 import fluid as F

    pos, rows = particles()
    f = _fluid(pos, rows)
    f.step_stages(DT, 0, 1)
    marker = f.download_grid(F.TAP_MARKER)
    taps = (F.TAP_UX, F.TAP_UY, F.TAP_UZ)
    for c in range(3):
        u = f.download_grid(taps[c])
        num, den = p2g_reference(pos, rows, c)
        ax = 2 - c
        nb = np.roll(marker, -1, axis=ax)
        face = ((marker == 1) | (nb == 1)) & (marker != 0) & (nb != 0)
        sl = [slice(None)] * 3
        sl[ax] = slice(0, -1)
        face_in = np.zeros_like(face)
        face_in[tuple(sl)] = face[tuple(sl)]
        with np.errstate(divide="ignore", invalid="ignore"):
            v = (num.astype(np.float64) / 2.0 ** 36) / (den.astype(np.float64) / 2.0 ** 40)
        want = np.where(den > 0, v.astype(np.float32), np.float32(0.0)) + np.float32(0.0)
        assert face_in.sum() > 5000 and (den[face_in] > 0).sum() > 5000
        same = (u.view(np.int32) == want.view(np.int32)) | (np.isnan(u) & np.isnan(want))
        bad = np.nonzero(face_in & ~same)
        assert bad[0].size == 0, f"u[{c}]: {bad[0].size} faces differ, first at (z, y, x) = {[int(b[0]) for b in bad]}"
