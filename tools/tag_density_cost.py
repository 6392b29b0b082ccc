"""What liquids of different densities cost on dam_256 (256^3 grid, 16.4 M particles).  Run from the repository root after
python -m blub_b200.build:

    python tools/tag_density_cost.py [--out profiles/h100_tag_density.json] [--rounds 3] [--steps 60]

  steps/s    dam_256 from the scene, the same step range [first, first + steps) with no table (default solver and path 6), a table of ones (tag 0 at 1.0) and half the
             liquid (the particles above the median height) tagged 1 at 0.8; the three in alternating rounds, device time from CUDA events
  stages     stage 0 and stage 2 of step_timed at the end of each timed range
  kernels    the cell-density kernels and the weighted solve kernel from torch.profiler over 5 eager steps of the half-tagged fluid, against
             the column solver's kernel of the fluid without a table over the same steps
Writes directories and files only at --out; reads the card name and power limit in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from blub_b200 import fluid as F  # noqa: E402
from tests import util  # noqa: E402

DT = F.DT_120HZ
CASES = ("none", "none_path6", "ones", "half_0.8")  # none_path6: no table on solver path 6, the tile kernel the weighted solve builds on


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def make(scene, case):
    f = blub_b200.HybridFluid.from_scene(scene)
    if case == "none_path6":
        f.set_solver_path(6)
    if case == "ones":
        f.set_tag_densities({0: 1.0})
    elif case == "half_0.8":
        pos = f.download_particles()
        pos[:, 3] = np.where(pos[:, 1] > np.median(pos[:, 1]), np.uint32(1), np.uint32(0)).view(np.float32)
        f.set_particles(pos)
        f.set_tag_densities({1: 0.8})
    return f


def timed(scene, case, first, steps):
    f = make(scene, case)
    for _ in range(first):
        f.step(DT)
    f.synchronize()
    stream = torch.cuda.ExternalStream(f.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        f.step(DT)
    e1.record(stream)
    e1.synchronize()
    ms = f.step_timed(DT)
    return steps / (e0.elapsed_time(e1) / 1000.0), ms[0], ms[2]


def kernels(scene, case, first):
    f = make(scene, case)
    for _ in range(first):
        f.step(DT)
    f.set_graph_replay(False)
    f.step(DT)
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(5):
            f.step(DT)
        f.synchronize()
    out = {}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for key in ("tag_density_scatter_kernel", "tag_density_finish_kernel", "tag_density_coeff_kernel", "pcg_solve_weighted_kernel",
                    "pcg_solve_columns_kernel", "pcg_solve_persistent_kernel"):
            if key in e.name:
                out.setdefault(key, []).append(round(e.device_time_total, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_tag_density.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--first", type=int, default=30)
    ap.add_argument("--steps", type=int, default=60)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    out = {"card": card(), "workload": "dam_256", "dt": DT, "step_range": [args.first, args.first + args.steps], "cases": list(CASES)}
    rates, st0, st2 = ({c: [] for c in CASES} for _ in range(3))
    for _ in range(args.rounds):
        for c in CASES:
            r, a, b = timed(scene, c, args.first, args.steps)
            rates[c].append(round(r, 2))
            st0[c].append(round(a, 3))
            st2[c].append(round(b, 3))
            print(c, rates[c][-1], st0[c][-1], st2[c][-1], flush=True)
    out["steps_per_s"] = rates
    out["stage0_ms"] = st0
    out["stage2_ms"] = st2
    out["kernel_us_per_launch"] = {c: kernels(scene, c, args.first) for c in ("half_0.8", "none", "none_path6")}
    out["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
