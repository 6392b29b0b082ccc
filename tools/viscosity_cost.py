"""What viscosity costs on dam_256 (256^3 grid, 16.4 M particles): steps/s of a fluid without viscosity and of fluids with k = nu dt of 0.1, 1
and 10, 3 x 100 steps each on the same step ranges, alternating in one process (the order alternates too); iterations per solve over 20 further
steps; whether a twin of the k = 1 fluid ends bit-identical; and, in a run of its own under torch.profiler (eager steps), the device time per
step of the set-up and solve kernels and the solve's time per iteration.  Reads the card name and power limit in the same run.  Run from the
repository root after python -m blub_b200.build:

    python tools/viscosity_cost.py [--out profiles/h100_viscosity.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from tests import util  # noqa: E402

DT = util.DT
NAMES = ("viscosity_setup_kernel", "viscosity_list_kernel", "viscosity_solve_kernel")
# the solve's loads and stores per live face and iteration (DESIGN.md §8 "Viscous liquids"): s . A s reads s and up to 6 neighbours (7 x 4 B),
# the update reads them again, reads and writes u and r (11 x 4 B), the new direction reads r and s and writes s (3 x 4 B); the cell's code
# word (4 B for its three faces) is read in each of the three passes
BYTES_PER_FACE_ITERATION = (7 + 11 + 3) * 4 + 3 * 4 / 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def profile_steps(f, steps=10):
    f.set_graph_replay(False)
    f.step(DT)
    f.synchronize()
    iterations = []
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(steps):
            f.step(DT)
            iterations.append(f.last_viscosity_solve()[0])
    per = {k: 0.0 for k in NAMES}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k in NAMES:
                if k in e.name:
                    per[k] += e.device_time_total
    ms = {k: round(v / steps / 1000, 4) for k, v in per.items()}
    marker = f.download_grid(blub_b200.fluid.TAP_MARKER)
    fluid_cells = int((marker == 1).sum())
    it = sum(iterations) / steps
    us_per_iteration = 1000 * ms["viscosity_solve_kernel"] / max(it, 1e-9)
    return {"device_ms_per_step": ms, "iterations_per_solve": it, "solve_us_per_iteration": round(us_per_iteration, 2), "fluid_cells": fluid_cells,
            "bytes_per_face_iteration": BYTES_PER_FACE_ITERATION,
            "solve_gb_per_s_on_3_faces_per_fluid_cell": round(3 * fluid_cells * BYTES_PER_FACE_ITERATION / (us_per_iteration * 1e-6) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_viscosity.json"))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    dt32 = float(np.float32(DT))
    fluids = {"k_0": blub_b200.HybridFluid.from_scene(scene)}
    for k in (0.1, 1.0, 10.0):
        fluids[f"k_{k:g}"] = blub_b200.HybridFluid.from_scene(scene)
        fluids[f"k_{k:g}"].set_viscosity(k / dt32)
    twin = blub_b200.HybridFluid.from_scene(scene)
    twin.set_viscosity(1.0 / dt32)
    for f in list(fluids.values()) + [twin]:
        f.step(DT)  # step 0 (rebinning) and the graph captures
        f.time_steps(DT, 9)
    rates = {k: [] for k in fluids}
    for r in range(args.rounds):
        for name, f in (list(fluids.items()) if r % 2 == 0 else list(fluids.items())[::-1]):
            rates[name].append(round(args.steps / (f.time_steps(DT, args.steps) / 1000.0), 2))
        twin.time_steps(DT, args.steps)
    same = bool(np.array_equal(twin.download_particles().view(np.uint32), fluids["k_1"].download_particles().view(np.uint32)))
    del twin
    iterations = {}
    for name, f in fluids.items():
        if name == "k_0":
            continue
        its = []
        for _ in range(20):
            f.step(DT)
            its.append(f.last_viscosity_solve()[0])
        iterations[name] = {"min": min(its), "median": statistics.median(its), "max": max(its)}
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": fluids["k_0"].num_particles,
        "dt": dt32,
        "steps_per_round": args.steps,
        "steps_per_s": rates,
        "iterations_per_solve": iterations,
        "twin_of_k_1_bit_identical": same,
        "profile_k_1": profile_steps(fluids["k_1"]),
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
