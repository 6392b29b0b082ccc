"""What CFL-limited substeps measure and cost on dam_256 (256^3 grid, 16.4 M particles, 0.005 m cells).  Run from the repository root after
python -m blub_b200.build:

    python tools/cfl_cost.py [--out profiles/h100_cfl.json]

  kernel      max_particle_velocity_kernel at 16.4 M particles: device time per launch from torch.profiler over 100 launches, and CUDA events
              around 100 consecutive blub_fluid_max_particle_velocity calls (each a kernel, a 12-byte read-back and a synchronise); 48 B per
              particle over the kernel time against the 3.35 TB/s of the H100 SXM data sheet
  overhead    advance() over 12 intervals of 1/120 s at C = 1 from rest, against replaying its dt list with plain steps on a fresh fluid,
              alternating 3 times in this process: ms per substep of each, and the difference
  runs        1 s simulated from rest at the fixed 1/120 s step and at C = 1: the largest per-axis particle velocity x dt after every
              step, substeps per interval, wall seconds per simulated second, both solves' iterations and final errors per step, and the
              most particles in one cell at t = 56/120 s
Reads the card name and power limit in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from blub_b200 import fluid as F  # noqa: E402
from tests import util  # noqa: E402

INTERVAL_NS = 8_333_333
BYTES_PER_PARTICLE = 48  # three velocity rows, one float4 each
HBM_TB_S = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def secs(dt_ns):
    return float(F.lib().blub_duration_as_secs_f32(int(dt_ns)))


def fresh(scene):
    f = blub_b200.HybridFluid.from_scene(scene)
    f.synchronize()
    return f


def kernel_time(scene, launches=100):
    f = fresh(scene)
    for _ in range(30):
        f.step()
    f.max_particle_velocity()  # warm-up: module load, allocation
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(launches):
            f.max_particle_velocity()
    times = [e.device_time_total for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "max_particle_velocity_kernel" in e.name]
    stream = torch.cuda.ExternalStream(f.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(launches):
        f.max_particle_velocity()
    e1.record(stream)
    e1.synchronize()
    call_ms = e0.elapsed_time(e1) / launches
    n = f.num_particles
    us = statistics.median(times)
    return {"particles": n, "launches_profiled": len(times), "kernel_us_median": round(us, 2), "kernel_us_min": round(min(times), 2),
            "kernel_us_max": round(max(times), 2), "call_ms_events": round(call_ms, 4),
            "bytes": n * BYTES_PER_PARTICLE, "tb_per_s": round(n * BYTES_PER_PARTICLE / (us * 1e-6) / 1e12, 3),
            "share_of_3_35_tb_s": round(n * BYTES_PER_PARTICLE / (us * 1e-6) / 1e12 / HBM_TB_S, 3)}


def overhead(scene, intervals=12, rounds=3):
    res = {"advance_ms_per_substep": [], "replay_ms_per_substep": [], "substeps": None}
    for _ in range(rounds):
        a = fresh(scene)
        t0 = time.perf_counter()
        plans = []
        for _ in range(intervals):
            plans += a.advance(INTERVAL_NS, cfl=1.0)
        a.synchronize()
        ta = time.perf_counter() - t0
        dts = [dt for dt, _ in plans]
        b = fresh(scene)
        t0 = time.perf_counter()
        for dt in dts:
            b.step(secs(dt))
        b.synchronize()
        tb = time.perf_counter() - t0
        same = bool(np.array_equal(a.download_particles().view(np.uint32), b.download_particles().view(np.uint32)))
        res["advance_ms_per_substep"].append(round(1000 * ta / len(dts), 3))
        res["replay_ms_per_substep"].append(round(1000 * tb / len(dts), 3))
        res["substeps"] = len(dts)
        res.setdefault("bit_identical", []).append(same)
        del a, b
    res["overhead_ms_per_substep"] = [round(x - y, 3) for x, y in zip(res["advance_ms_per_substep"], res["replay_ms_per_substep"])]
    return res


def most_in_one_cell(f):
    p = f.download_particles()[:, :3]
    c = np.clip(np.floor(p).astype(np.int64), 0, [f.nx - 1, f.ny - 1, f.nz - 1])
    return int(np.bincount((c[:, 2] * f.ny + c[:, 1]) * f.nx + c[:, 0]).max())


def new_solves(f, k):
    """both solves of the last k steps: [(iterations, error)] from the solver statistics (error = max |r| * dt)"""
    f.synchronize()
    f.update_statistics()
    return [f.pressure_solver_stats(w)[-k:] for w in (0, 1)]


def summary(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs)} if xs else None


def run(scene, cfl, seconds=1.0):
    f = fresh(scene)
    per_step, per_interval, solves, crowd = [], [], [[], []], None
    t0 = time.perf_counter()
    for i in range(int(round(seconds * 120))):
        if cfl is None:
            f.step(secs(INTERVAL_NS))
            v = f.max_particle_velocity()
            per_step.append({"dt_ns": INTERVAL_NS, "cells": [x * secs(INTERVAL_NS) for x in v]})
            k = 1
        else:
            plans = f.advance(INTERVAL_NS, cfl=cfl)
            # the velocity after each substep is the one the next plan measured; the last one is measured here
            after = [v for _, v in plans[1:]] + [f.max_particle_velocity()]
            per_step += [{"dt_ns": dt, "cells": [x * secs(dt) for x in v]} for (dt, _), v in zip(plans, after)]
            k = len(plans)
        per_interval.append(k)
        for w, s in enumerate(new_solves(f, min(k, 100))):
            solves[w] += s
        if i + 1 == 56:
            crowd = most_in_one_cell(f)
    wall = time.perf_counter() - t0
    worst = [max(s["cells"]) for s in per_step]
    return {
        "cfl": cfl, "steps": len(per_step), "substeps_per_interval": summary(per_interval), "wall_s_per_simulated_s": round(wall / seconds, 3),
        "max_axis_cells_per_step": {"max": round(max(worst), 3), "median": round(statistics.median(worst), 3),
                                    "after_step": [round(x, 3) for x in worst]},
        "most_particles_in_one_cell_at_56_120_s": crowd,
        "solves": {name: {"iterations": summary([it for _, it in solves[w]]), "final_error_max_r_dt": summary([float(e) for e, _ in solves[w]]),
                          "samples": len(solves[w])} for w, name in enumerate(("velocity", "density"))},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_cfl.json"))
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    out = {"card": card(), "workload": "dam_256", "interval_ns": INTERVAL_NS}
    out["kernel"] = kernel_time(scene)
    print(json.dumps(out["kernel"]), flush=True)
    out["overhead"] = overhead(scene)
    print(json.dumps(out["overhead"]), flush=True)
    out["fixed_120hz"] = run(scene, None)
    out["cfl_1"] = run(scene, 1.0)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k not in ("fixed_120hz", "cfl_1")}))
    for k in ("fixed_120hz", "cfl_1"):
        print(k, json.dumps({a: b for a, b in out[k].items() if a != "max_axis_cells_per_step"}), out[k]["max_axis_cells_per_step"]["max"])


if __name__ == "__main__":
    main()
