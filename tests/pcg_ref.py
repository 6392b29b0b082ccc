"""Float64 restatement of the pressure solve (pcg.cu, DESIGN §3.1), one iteration at a time, with a bound for every element the kernels
round.  NumPy only; independent of the oracle.  Volumes are [z, y, x].

The solve, as the kernels compute it:
  * codes: diag = the number of non-SOLID neighbours (bits 0..2), the FLUID bit; p, r, s are exactly 0 off FLUID (the zero invariant);
  * A x = diag x - (sum of the six neighbours) on FLUID cells, 0 elsewhere;
  * z = r c_inv_diag2[diag] (precond_mode 0; the table's float32 constants taken as exact), or the literal two passes of precond_mode 1:
    t = (r - r[-x] - r[-y] - r[-z]) / diag, z = (t - t[-x] - t[-y] - t[-z]) / diag (no division where diag = 0);
  * init: r_0 = b - A p_0, sigma_0 = z_0 . r_0, s_{-1} = 0, beta_{-1} = 0;
  * iteration k: s_k = z_k + beta_{k-1} s_{k-1}; alpha_k = guarded_div(sigma_k, s_k . A s_k); p_{k+1} = p_k + alpha_k s_k;
    r_{k+1} = r_k - alpha_k A s_k; sigma_{k+1} = z_{k+1} . r_{k+1}; beta_k = guarded_div(sigma_{k+1}, sigma_k);
  * the stop test at i == max or (i > 0 and i % freq == 0): max|r_{i+1}| < error_tolerance / dt (float32).

Observation protocol.  A solve with tolerance 0 and max_num_iterations = K stops after iteration K and leaves p_{K+1}, r_{K+1}, the
scalars of iteration K and max|r_{K+1}|.  Runs K = 0, 1, ... from the same p_0 and b are prefixes of each other, so every iterate and
every scalar the solver used is observed, and each check below is ONE step from an observed state: r_k (k >= 1) and p_k are the float32
arrays of run k - 1, alpha, beta and sigma the float32 values of the runs.  s_k is not observed: it is carried as a float64 recursion
from the observed r_k and beta, with its own bound.

Bounds: first-order propagation of u = 2^-24 per rounding times the magnitude of the rounded result,
    a +- b: e_a + e_b + u |a +- b|        a b: |b| e_a + |a| e_b + u |a b|        a / b: (e_a + |a / b| e_b) / |b| + u |a / b|
A contracted FMA rounds once where the separate operations round twice, and the dropped rounding is one of the terms above: every bound
holds with and without FMA contraction.  Sums of n float32 terms are bounded by (depth) u sum|terms|, with the depth the longest chain
of float32 additions any term passes through:
  * the stencil: depth 7 over d|x| + sum|x_nbr| (the kernels' tree has depth 4; the oracle subtracts the neighbours one by one);
  * r_0 = b - A p_0: depth 8 over |b| + d|p_0| + sum|p_0 nbr|;
  * the dot products (REDUCTIONS): a thread adds its quads' pairs (2 levels) to its accumulator in every pass over 4 planes, the block
    adds 32 lanes by shuffles (5 levels) and 8 warps (3 tree levels in block_sum, 8 in sequence in the column solver's reducer), then
    the blocks' partials are added in fp64 and rounded once to float32; the oracle adds 16 strided terms, then a 1024-wide tree, per
    level of its multi-pass reduction.
guarded_div is emulated exactly in float32 (IEEE division: nvcc's default -prec-div=true).  Every bound is multiplied by 1.001
(second-order terms) and 1e-30 is added (denormals).  Nothing is fitted to data.
"""
import numpy as np

SOLID, FLUID, AIR = 0, 1, -1
U = 2.0 ** -24
SAFETY = 1.001
TINY = 1e-30
f32 = np.float32
PCG_EPSILON = f32(1e-10)
C_INV_DIAG2 = np.array([1.0, 1.0, 0.25, 1.0 / 9.0, 0.0625, 0.04, 1.0 / 36.0, 1.0], dtype=f32)
STENCIL_DEPTH = 7
INIT_DEPTH = 8


class Mismatch(AssertionError):
    """An element outside its bound (or not bit-identical where it must be), named."""


# ------------------------------------------------------------------------------------------------ the system
def system(m):
    """(diag, fluid) of a marker: diag = number of non-SOLID neighbours, the border counts as SOLID.  No FLUID cell on the border."""
    m = np.asarray(m)
    fl = m == FLUID
    assert not (fl[0].any() or fl[-1].any() or fl[:, 0].any() or fl[:, -1].any() or fl[:, :, 0].any() or fl[:, :, -1].any()), \
        "FLUID on the border"
    ns = np.pad(m != SOLID, 1).astype(np.int64)
    diag = (ns[:-2, 1:-1, 1:-1] + ns[2:, 1:-1, 1:-1] + ns[1:-1, :-2, 1:-1] + ns[1:-1, 2:, 1:-1] + ns[1:-1, 1:-1, :-2] + ns[1:-1, 1:-1, 2:])
    return diag, fl


def nbr_sum(x):
    p = np.pad(x, 1)
    return p[:-2, 1:-1, 1:-1] + p[2:, 1:-1, 1:-1] + p[1:-1, :-2, 1:-1] + p[1:-1, 2:, 1:-1] + p[1:-1, 1:-1, :-2] + p[1:-1, 1:-1, 2:]


def lower_sum(x):
    """x[-x] + x[-y] + x[-z] (the neighbours the literal preconditioner passes read)."""
    p = np.pad(x, ((1, 0), (1, 0), (1, 0)))
    return p[:-1, 1:, 1:] + p[1:, :-1, 1:] + p[1:, 1:, :-1]


def apply_A(diag, fl, x):
    """(A x, depth-free magnitude d|x| + sum|x_nbr|) on FLUID cells, 0 elsewhere; x must be 0 off FLUID."""
    v = np.where(fl, diag * x - nbr_sum(x), 0.0)
    mag = np.where(fl, diag * np.abs(x) + nbr_sum(np.abs(x)), 0.0)
    return v, mag


def guarded_div(num, den):
    """guarded_div of pcg.cu in float32: num / (den + (den < 0 ? -eps : eps))."""
    num, den = f32(num), f32(den)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return f32(num / f32(den + (-PCG_EPSILON if den < 0 else PCG_EPSILON)))


# ------------------------------------------------------------------------------------------------ (value, bound) steps
def precondition(diag, fl, r, er, mode=0, z_roundings=1):
    """z = M^-1 r with its bound.  mode 0: r c_inv_diag2[d] (z_roundings = 1: the table; 3: (r / d) / d as the oracle divides, which
    also differs from the table's rounded constant by u |z|).  mode 1: the two literal passes."""
    if mode == 0:
        c = C_INV_DIAG2[np.minimum(diag, 7)].astype(np.float64)
        z = np.where(fl, r * c, 0.0)
        return z, np.where(fl, c * er + z_roundings * U * np.abs(z), 0.0)
    dd = np.maximum(diag, 1).astype(np.float64)
    div = (diag > 1).astype(np.float64)  # a division by 1 is exact
    out, eo = r, er
    for _ in range(2):
        t = np.where(fl, (out - lower_sum(out)) / dd, 0.0)
        et = np.where(fl, (eo + lower_sum(eo) + 3 * U * (np.abs(out) + lower_sum(np.abs(out)))) / dd + div * U * np.abs(t), 0.0)
        out, eo = t, et
    return out, eo


def stencil(diag, fl, s, es):
    As, mag = apply_A(diag, fl, s)
    return As, np.where(fl, diag * es + nbr_sum(es) + STENCIL_DEPTH * U * mag, 0.0)


class Reduction:
    """How a dot product is summed: `depth` float32 addition levels over sum|terms|, then (fp64 = number of fp64 partials, or 0) the
    blocks' partials in fp64 and one rounding to float32."""

    def __init__(self, depth, fp64=0, name=""):
        self.depth, self.fp64, self.name = depth, fp64, name

    def bound(self, abs_sum, value):
        e = self.depth * U * abs_sum
        if self.fp64:
            e = e + self.fp64 * 2.0 ** -53 * abs_sum + U * abs(value)
        return e


def slab_reduction(passes, world):
    """The z-slab ranks: every rank's blocks as gpu_reduction, its total rounded to float32 once for the mailbox (one more level), the
    ranks' totals added in fp64 and rounded once."""
    r = gpu_reduction(passes)
    return Reduction(r.depth + 1, fp64=r.fp64 * world + world, name=f"slab({passes} passes, {world} ranks)")


def gpu_reduction(passes, column_reducer=True):
    """A thread's `passes` tile / column passes of 4 planes each, its quad pairs (2 levels), 5 shuffle levels and the 8 warps (8 in
    sequence or a 3-level tree), then fp64 over at most 4096 blocks."""
    return Reduction(2 + 4 * passes + 5 + (8 if column_reducer else 3), fp64=4096, name=f"gpu({passes} passes)")


def oracle_reduction(n):
    """oracle reduce_all: while more than 16384 values remain a strided pass (16 terms in sequence + a 10-level tree), then one group."""
    levels, rem = 1, n
    while rem > 16384:
        rem = (rem // 16 + 1023) // 1024
        levels += 1
    return Reduction(26 * levels, name=f"oracle({levels} levels)")


def dot(x, ex, y, ey, red):
    """sum x y with its bound (products rounded once, then summed as `red` does)."""
    v = float(np.sum(x * y))
    a = float(np.sum(np.abs(x * y)))
    e = float(np.sum(np.abs(y) * ex + np.abs(x) * ey)) + U * a + red.bound(a, v)
    return v, e


# ------------------------------------------------------------------------------------------------ observations
class Run:
    """What one solve with tolerance 0 and max_num_iterations = K leaves."""

    def __init__(self, p, r, scalars, max_error, iterations):
        self.p = np.asarray(p, dtype=f32)
        self.r = np.asarray(r, dtype=f32)
        self.alpha, self.beta, self.sigma = (f32(v) for v in scalars)
        self.max_error = f32(max_error)
        self.iterations = int(iterations)


def scalar_tables(runs, convention):
    """alpha[k], beta[k] (beta_k: forms s_{k+1}), sigma[k] from the runs.  convention "persistent": run K leaves (alpha_K, beta_{K-1},
    sigma_K); "update" (three-kernel path, precond_mode 0): (alpha_K, beta_K, sigma_{K+1})."""
    alpha, beta, sigma = {}, {}, {}
    for K, run in enumerate(runs):
        alpha[K] = run.alpha
        if convention == "persistent":
            beta[K - 1], sigma[K] = run.beta, run.sigma
        else:
            assert convention == "update", convention
            beta[K], sigma[K + 1] = run.beta, run.sigma
    return alpha, beta, sigma


class Stats:
    """Observed error / bound per quantity, for the report."""

    def __init__(self):
        self.ratios = {}

    def add(self, what, ratio):
        self.ratios.setdefault(what, []).append(np.atleast_1d(np.asarray(ratio, dtype=np.float64)).ravel())

    def summary(self):
        out = {}
        for k, v in self.ratios.items():
            a = np.concatenate(v)
            out[k] = (float(np.median(a)), float(a.max())) if a.size else (0.0, 0.0)
        return out

    def line(self):
        return ", ".join(f"{k} {med:.2e} / {mx:.2e}" for k, (med, mx) in self.summary().items())


def _where(shape, flat):
    z, y, x = np.unravel_index(int(flat), shape)
    return f"cell (x={x}, y={y}, z={z})"


def check_elements(label, k, what, obs, ref, bound, fl, stats):
    """FLUID cells within their bound, every other cell exactly 0."""
    obs64 = obs.astype(np.float64)
    off = ~fl & (obs != 0)
    if off.any():
        i = np.flatnonzero(off)[0]
        raise Mismatch(f"{label}: iteration {k}, {what} at {_where(obs.shape, i)} (not FLUID): observed {obs.ravel()[i]!r}, must be 0")
    b = SAFETY * bound + TINY
    d = np.abs(obs64 - ref)
    bad = fl & ~(d <= b)
    if bad.any():
        i = int(np.argmax(np.where(bad, d / b, -1.0).ravel()))
        raise Mismatch(f"{label}: iteration {k}, {what} at {_where(obs.shape, i)}: observed {obs64.ravel()[i]!r}, reference "
                       f"{ref.ravel()[i]!r}, |difference| {d.ravel()[i]:.3e} > bound {b.ravel()[i]:.3e}")
    if fl.any():
        stats.add(what, d[fl] / b[fl])


def check_scalar(label, k, what, obs, ref, bound, stats):
    b = SAFETY * bound + TINY
    d = abs(float(obs) - ref)
    if not d <= b:
        raise Mismatch(f"{label}: iteration {k}, {what}: observed {float(obs)!r}, reference {ref!r}, |difference| {d:.3e} > bound {b:.3e}")
    stats.add(what, d / b)


def check_runs(label, m, b, p0, runs, red, convention="persistent", mode=0, z_roundings=1, stats=None):
    """Every run K of `runs` (runs[K] stopped after iteration K) one step from the observed state of run K - 1 (module docstring).
    Raises Mismatch naming the first element outside its bound.  Returns the Stats."""
    stats = Stats() if stats is None else stats
    diag, fl = system(m)
    shape = diag.shape
    alpha, beta, sigma = scalar_tables(runs, convention)
    if convention == "persistent" and runs and runs[0].beta != 0:
        raise Mismatch(f"{label}: iteration 0, beta_-1: observed {float(runs[0].beta)!r}, must be 0")
    b64 = np.where(fl, np.asarray(b, dtype=np.float64), 0.0)
    p = np.where(fl, np.asarray(p0, dtype=np.float64), 0.0)
    Ap, mag = apply_A(diag, fl, p)
    r = np.where(fl, b64 - Ap, 0.0)
    er = np.where(fl, INIT_DEPTH * U * (np.abs(b64) + mag), 0.0)
    s_prev, es_prev = np.zeros(shape), np.zeros(shape)
    zr_prev = ezr_prev = 0.0
    for k, run in enumerate(runs):
        if k > 0:
            p = runs[k - 1].p.astype(np.float64)
            r = runs[k - 1].r.astype(np.float64)
            er = np.zeros(shape)
        z, ez = precondition(diag, fl, r, er, mode, z_roundings)
        zr, ezr = dot(z, ez, r, er, red)
        if k in sigma:
            check_scalar(label, k, "sigma", sigma[k], zr, ezr, stats)
        if k >= 1 and k in sigma and k - 1 in sigma and k - 1 in beta:
            want = guarded_div(sigma[k], sigma[k - 1])
            if beta[k - 1].tobytes() != want.tobytes():
                raise Mismatch(f"{label}: iteration {k}, beta_{k - 1}: observed {float(beta[k - 1])!r}, guarded_div(sigma_{k}, sigma_{k - 1}) "
                               f"= {float(want)!r}")
        elif k >= 1 and k in sigma and k - 1 in beta and abs(zr_prev) > ezr_prev:
            # sigma_{k-1} not observed ("update": sigma_0): beta_{k-1} against sigma_k / (the reference's sigma_{k-1} +- eps)
            g = float(PCG_EPSILON) if zr_prev > 0 else -float(PCG_EPSILON)
            want = float(sigma[k]) / (zr_prev + g)
            check_scalar(label, k, f"beta_{k - 1}", beta[k - 1], want, abs(want) * ezr_prev / abs(zr_prev + g) + 2 * U * abs(want), stats)
        zr_prev, ezr_prev = zr, ezr
        bk = float(beta[k - 1]) if k >= 1 else 0.0
        s = np.where(fl, z + bk * s_prev, 0.0)
        es = np.where(fl, ez + abs(bk) * es_prev + U * np.abs(bk * s_prev) + U * np.abs(s), 0.0)
        As, eAs = stencil(diag, fl, s, es)
        den, eden = dot(s, es, As, eAs, red)
        a = float(alpha[k])
        if k in sigma:
            sg = float(sigma[k])
            if sg == 0.0:
                if a != 0.0:
                    raise Mismatch(f"{label}: iteration {k}, alpha: observed {a!r} with sigma = 0, must be 0")
            else:
                used = sg / a  # the guarded s.As the solver divided by, up to two roundings
                # the guard's sign follows the sign of the float32 s.As: known unless the reference is within its bound of 0
                signs = [1.0] if den - eden > 0 else ([-1.0] if den + eden < 0 else [1.0, -1.0])
                d = min(abs(used - sg_ * float(PCG_EPSILON) - den) for sg_ in signs)
                bnd = SAFETY * (eden + 2 * U * abs(used)) + TINY
                if not d <= bnd:
                    raise Mismatch(f"{label}: iteration {k}, s.As (sigma / alpha = {used!r}): reference {den!r}, |difference| {d:.3e} > bound {bnd:.3e}")
                stats.add("s.As", d / bnd)
        elif abs(zr) > ezr and abs(den) > eden:
            # sigma_k not observed ("update": sigma_0): alpha_k against guarded_div of the reference's sigma_k and s.As
            g = float(PCG_EPSILON) if den > 0 else -float(PCG_EPSILON)
            want = zr / (den + g)
            check_scalar(label, k, "alpha", alpha[k], want, abs(want) * (ezr / abs(zr) + eden / abs(den + g)) + 2 * U * abs(want), stats)
        p_ref = p + a * s
        ep = np.abs(a) * es + U * np.abs(a * s) + U * np.abs(p_ref)
        r_ref = r - a * As
        er_new = er + abs(a) * eAs + U * np.abs(a * As) + U * np.abs(r_ref)
        check_elements(label, k, "p", run.p, p_ref, ep, fl, stats)
        check_elements(label, k, "r", run.r, r_ref, er_new, fl, stats)
        mx = f32(np.abs(run.r).max()) if run.r.size else f32(0)
        if run.max_error.tobytes() != mx.tobytes():
            raise Mismatch(f"{label}: iteration {k}, max|r|: observed {float(run.max_error)!r}, max|r_{k + 1}| = {float(mx)!r}")
        if run.iterations != k:
            raise Mismatch(f"{label}: iteration {k}, iteration count {run.iterations}")
        s_prev, es_prev = s, es
    return stats


# ------------------------------------------------------------------------------------------------ the stop schedule
def tolerance32(error_tolerance, dt):
    """The solver's float32 threshold: error_tolerance / dt with both in float32."""
    return f32(f32(error_tolerance) / f32(dt))


def predict_stop(maxima, tol, freq, max_it):
    """First iteration i at which a solve with this schedule stops; maxima[i] = max|r_{i+1}| observed after iteration i."""
    for i in range(max_it + 1):
        if i == max_it or (i > 0 and i % freq == 0 and f32(maxima[i]) < f32(tol)):
            return i
    raise AssertionError("unreachable")


def tolerance_between(maxima, lo_it, hi_it, dt):
    """An error_tolerance whose float32 threshold lies strictly between maxima[hi_it] and maxima[lo_it], far from both (geometric mean)."""
    hi, lo = float(maxima[lo_it]), float(maxima[hi_it])
    assert lo < hi, (lo_it, hi_it, lo, hi)
    tol = float(f32(np.sqrt(hi * lo) * dt))
    t32 = tolerance32(tol, dt)
    assert lo < t32 < hi
    return tol


# ------------------------------------------------------------------------------------------------ plain float64 PCG (closed forms)
def cg64(m, b, p0, iterations, mode=0):
    """The recurrence in float64 with the table's constants: [(p_{k+1}, r_{k+1}, alpha_k, beta_{k-1}, sigma_k)] for k < iterations."""
    diag, fl = system(m)
    zero = np.zeros(diag.shape)
    p = np.where(fl, np.asarray(p0, dtype=np.float64), 0.0)
    r = np.where(fl, np.asarray(b, dtype=np.float64), 0.0) - apply_A(diag, fl, p)[0]
    z = precondition(diag, fl, r, zero, mode)[0]
    sigma, beta, s = float(np.sum(z * r)), 0.0, zero
    eps = float(PCG_EPSILON)
    out = []
    for k in range(iterations):
        s = z + beta * s
        As = apply_A(diag, fl, s)[0]
        den = float(np.sum(s * As))
        alpha = sigma / (den + (-eps if den < 0 else eps))
        p = p + alpha * s
        r = r - alpha * As
        out.append((p.copy(), r.copy(), alpha, beta, sigma))
        z = precondition(diag, fl, r, zero, mode)[0]
        zr = float(np.sum(z * r))
        beta = zr / (sigma + (-eps if sigma < 0 else eps))
        sigma = zr
    return out


# ------------------------------------------------------------------------------------------------ a float32 emulation (mutants)
def emulate32(m, b, p0, iterations, mode=0, block=64, mutation=None):
    """The solve in float32 NumPy with the persistent solvers' conventions: the runs K = 0 .. iterations - 1.  Partial sums over blocks of
    `block` consecutive cells are rounded to float32 and added in fp64, then rounded once (Reduction(1, fp64)).  `mutation` = (name, k,
    arg) plants one defect at iteration k: "drop_neighbour" (A s at cell index arg leaves out its +x neighbour in the r update),
    "alpha_scale" (alpha_k times 1 + arg), "stale_beta" (beta_{k} formed from sigma_{k-1}), "c_inv_diag2" (table entry arg scaled by
    1 + 2^-10, every iteration), "drop_partial" (sigma_{k} without its largest block partial), "max_lanes" (max|r| leaves out the lane x % 4 == arg)."""
    name, km, arg = mutation if mutation else (None, -1, None)
    diag, fl = system(m)
    table = C_INV_DIAG2.copy()
    if name == "c_inv_diag2":
        table[arg] = f32(table[arg] * f32(1 + 2.0 ** -10))
    code_c = np.where(fl, table[np.minimum(diag, 7)], f32(0))
    d32 = diag.astype(f32)

    def red(t, drop=False):
        t = t.astype(f32).ravel()
        n = -(-t.size // block) * block
        parts = np.pad(t, (0, n - t.size)).astype(np.float64).reshape(-1, block).sum(axis=1).astype(f32)
        if drop:
            parts[np.abs(parts).argmax()] = 0
        return f32(parts.astype(np.float64).sum())

    def A(x, dropped=None):
        pz = np.pad(x, 1)
        xm, xp = pz[1:-1, 1:-1, :-2], pz[1:-1, 1:-1, 2:]
        if dropped is not None:
            xp = xp.copy()
            xp.ravel()[dropped] = 0
        s6 = ((xm + xp) + (pz[1:-1, :-2, 1:-1] + pz[1:-1, 2:, 1:-1])) + (pz[:-2, 1:-1, 1:-1] + pz[2:, 1:-1, 1:-1])
        return np.where(fl, d32 * x - s6, f32(0)).astype(f32)

    def prec(r):
        if mode == 0:
            return (r * code_c).astype(f32)
        dd = np.maximum(diag, 1).astype(f32)
        out = r
        for _ in range(2):
            pz = np.pad(out, ((1, 0), (1, 0), (1, 0)))
            out = np.where(fl, (out - ((pz[1:, 1:, :-1] + pz[1:, :-1, 1:]) + pz[:-1, 1:, 1:])) / dd, f32(0)).astype(f32)
        return out

    p = np.where(fl, np.asarray(p0, dtype=f32), f32(0)).astype(f32)
    r = np.where(fl, (np.asarray(b, dtype=f32) - A(p)), f32(0)).astype(f32)
    z = prec(r)
    sigma, beta, s = red(z * r, drop=name == "drop_partial" and km == 0), f32(0), np.zeros_like(r)
    sigma_prev = sigma
    lanes = np.ones(diag.shape, dtype=bool)
    if name == "max_lanes":
        lanes[:, :, arg::4] = False
    runs = []
    for k in range(iterations):
        s = (z + beta * s).astype(f32)
        den = red(s * A(s))
        alpha = guarded_div(sigma, den)
        if name == "alpha_scale" and k == km:
            alpha = f32(alpha * f32(1 + arg))
        p = (p + alpha * s).astype(f32)
        r = (r - alpha * A(s, arg if name == "drop_neighbour" and k == km else None)).astype(f32)
        runs.append(Run(p.copy(), r.copy(), (alpha, beta, sigma), np.abs(np.where(lanes, r, 0)).max(), k))
        z = prec(r)
        zr = red(z * r, drop=name == "drop_partial" and k + 1 == km)
        beta = guarded_div(zr, sigma_prev if name == "stale_beta" and k == km else sigma)
        sigma_prev, sigma = sigma, zr
    return runs
