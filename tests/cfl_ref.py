"""Python restatement of the CFL substep rule of blub_cfl_substep_ns (include/blub_fluid.h, DESIGN.md §8 "CFL-limited substeps").

Float64 for the speeds and the step in seconds, Python integers for nanoseconds.  Raises ValueError where the library returns
BLUB_ERR_INVALID_ARGUMENT and Unstable where it returns BLUB_ERR_UNSTABLE.
"""
import math

import numpy as np

U64_MAX = (1 << 64) - 1


class Unstable(Exception):
    pass


def check_config(cfl, max_dt_ns, min_dt_ns, reserved=0):
    c = float(np.float32(cfl))
    if not math.isfinite(c) or not (0.0 < c <= 16.0):
        raise ValueError("cfl_number must be finite and in (0, 16]")
    if reserved != 0:
        raise ValueError("reserved must be 0")
    if not (1 <= min_dt_ns <= max_dt_ns):
        raise ValueError("1 <= min_dt_ns <= max_dt_ns")
    return c


def cfl_step_ns(max_velocity, gravity, cfl, max_dt_ns):
    """d_ns: the CFL step before the min_dt_ns check and the split of the remaining time."""
    v = [float(np.float32(x)) for x in max_velocity]
    g = [float(np.float32(x)) for x in gravity]
    u = max(abs(x) for x in v)
    s = u + math.sqrt(5.0 * math.sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]))
    d = float(np.float32(cfl)) / s if s > 0.0 else math.inf
    scaled = d * 1e9
    if scaled >= 2.0 ** 64:
        return max_dt_ns
    return min(max_dt_ns, math.floor(scaled))


def substep_ns(remaining_ns, max_velocity, gravity, cfl, max_dt_ns, min_dt_ns, reserved=0):
    check_config(cfl, max_dt_ns, min_dt_ns, reserved)
    if remaining_ns == 0:
        raise ValueError("remaining_ns must be above 0")
    if not all(math.isfinite(float(np.float32(x))) for x in gravity):
        raise ValueError("gravity is not finite")
    if not all(math.isfinite(float(np.float32(x))) for x in max_velocity):
        raise Unstable("the largest particle velocity is not finite")
    d_ns = cfl_step_ns(max_velocity, gravity, cfl, max_dt_ns)
    if d_ns < min_dt_ns:
        raise Unstable(f"the CFL step of {d_ns} ns is below min_dt_ns = {min_dt_ns} ns")
    if remaining_ns <= d_ns:
        return remaining_ns
    if remaining_ns < 2 * d_ns:
        return remaining_ns - remaining_ns // 2
    return d_ns
