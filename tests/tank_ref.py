"""NumPy restatement of the moving-tank rules (DESIGN.md §8 "Moving tanks"): the step constants in float64, the CFL bound, and
tank_frame_kernel in float32 with the kernel's order of operations, so that the GPU rows can be compared bit for bit."""
import numpy as np


def skew(v):
    """[v]x: skew(v) @ r == cross(v, r)."""
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def rotation_about(n, theta):
    """Rot(n, theta) by Rodrigues' formula (n a unit vector)."""
    n = np.asarray(n, dtype=np.float64)
    return np.cos(theta) * np.eye(3) + np.sin(theta) * skew(n) + (1.0 - np.cos(theta)) * np.outer(n, n)


def step_constants(frame, gravity, dt):
    """float64 g_eff, Q, K and pivot of a frame dict for float32 gravity and the step's float32 dt (not yet rounded)."""
    R = np.asarray(frame["rotation"], dtype=np.float64).reshape(3, 3)
    g = np.asarray(gravity, dtype=np.float32).astype(np.float64)
    A = np.asarray(frame.get("acceleration", (0, 0, 0)), dtype=np.float64)
    w = np.asarray(frame.get("angular_velocity", (0, 0, 0)), dtype=np.float64)
    al = np.asarray(frame.get("angular_acceleration", (0, 0, 0)), dtype=np.float64)
    h = float(np.float32(dt))
    wn = float(np.linalg.norm(w))
    Q = rotation_about(w / wn, -2.0 * wn * h) if wn > 0 else np.eye(3)
    K = h * (np.dot(w, w) * np.eye(3) - np.outer(w, w) - skew(al))
    return {"gravity": R.T @ (g - A), "coriolis": Q, "force": K, "pivot": np.asarray(frame.get("pivot", (0, 0, 0)), dtype=np.float64)}


def cfl_inputs(max_velocity, gravity, frame, dims):
    """The (velocity, gravity) float32 triples blub_tank_cfl_substep_ns passes to the CFL rule under a frame."""
    if frame is None:
        return np.asarray(max_velocity, dtype=np.float32), np.asarray(gravity, dtype=np.float32)
    geff = step_constants(frame, gravity, 1.0)["gravity"].astype(np.float32).astype(np.float64)
    p = np.asarray(frame["pivot"], dtype=np.float64)
    corners = np.array([[(c >> k) & 1 for k in range(3)] for c in range(8)], dtype=np.float64) * np.asarray(dims, dtype=np.float64)
    r_max = np.sqrt(((corners - p) ** 2).sum(axis=1)).max()
    w = np.asarray(frame["angular_velocity"], dtype=np.float64)
    g = np.float32(np.sqrt((geff ** 2).sum()) + (np.dot(w, w) + np.linalg.norm(frame["angular_acceleration"])) * r_max)
    v = np.asarray(max_velocity, dtype=np.float32)
    if (w != 0).any():
        v = np.array([np.sqrt((v.astype(np.float64) ** 2).sum()), 0.0, 0.0], dtype=np.float32)
    return v, np.array([g, 0.0, 0.0], dtype=np.float32)


def apply_frame_kernel(pos, rows, coriolis, force, pivot):
    """tank_frame_kernel on float32 positions [n, 4] and rows [3, n, 4] with the library's float32 Q, K and pivot: every product and sum rounded
    to float32 in the kernel's order.  Returns the new rows."""
    f32 = np.float32
    q, k = np.asarray(coriolis, dtype=f32).reshape(3, 3), np.asarray(force, dtype=f32).reshape(3, 3)
    pv = np.asarray(pivot, dtype=f32)
    rows = np.asarray(rows, dtype=f32)
    r = [(pos[:, d] - pv[d]).astype(f32) for d in range(3)]
    out = np.empty_like(rows)
    with np.errstate(all="ignore"):
        for c in range(3):
            rot = ((q[c, 0] * rows[0]).astype(f32) + (q[c, 1] * rows[1]).astype(f32)).astype(f32)
            rot = (rot + (q[c, 2] * rows[2]).astype(f32)).astype(f32)
            f = ((k[c, 0] * r[0]).astype(f32) + (k[c, 1] * r[1]).astype(f32)).astype(f32)
            f = (f + (k[c, 2] * r[2]).astype(f32)).astype(f32)
            out[c, :, :3] = (rot[:, :3] + k[c][None, :]).astype(f32)
            out[c, :, 3] = (rot[:, 3] + f).astype(f32)
    return out
