"""What solid load probes cost on dam_256 (256^3 grid, 16.4 M particles): steps/s of a fluid without probes and of one with 6 probes (the four
side walls, the floor and one whole-grid probe), 3 x 100 steps each, alternating in one process (which fluid goes first alternates too),
with bit-identical particle output checked at the end; and the probe kernels' time per step with torch.profiler in a run of its own (the
slot clear and the box walk, every probe set in one launch pair), for the 6-probe set and for each probe alone.  Reads the card name and
power limit in the same run.  Run from the repository root after python -m blub_b200.build:

    python tools/load_cost.py [--out profiles/h100_loads.json]
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
from tests import util  # noqa: E402

DT = util.DT
N = 256
PROBES = {
    "wall_x0": ((0, 0, 0), (1, N, N)),
    "wall_x1": ((N - 1, 0, 0), (N, N, N)),
    "wall_z0": ((0, 0, 0), (N, N, 1)),
    "wall_z1": ((0, 0, N - 1), (N, N, N)),
    "floor": ((0, 0, 0), (N, 1, N)),
    "whole_grid": ((0, 0, 0), (N, N, N)),
}
KERNELS = ("solid_load_kernel", "load_slot_clear_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def kernel_ms_per_step(f, steps=10):
    """torch.profiler device time of the two probe kernels per step, over `steps` graph-replayed steps."""
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(steps):
            f.step(DT)
        f.synchronize()
    per = {k: 0.0 for k in KERNELS}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k in KERNELS:
                if k in e.name:
                    per[k] += e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_loads.json"))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    fluids = {"no_probes": blub_b200.HybridFluid.from_scene(scene), "six_probes": blub_b200.HybridFluid.from_scene(scene)}
    fluids["six_probes"].set_load_probes(list(PROBES.values()))
    for f in fluids.values():
        f.step(DT)  # step 0 (rebinning) and the graph captures
        f.time_steps(DT, 9)
    rates = {k: [] for k in fluids}
    for r in range(args.rounds):  # the same step range for both fluids; which one goes first alternates
        for name, f in (list(fluids.items()) if r % 2 == 0 else list(fluids.items())[::-1]):
            rates[name].append(round(args.steps / (f.time_steps(DT, args.steps) / 1000.0), 2))
    for f in fluids.values():
        f.synchronize()
    a, b = (fluids[k].download_particles() for k in ("no_probes", "six_probes"))
    same = a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
    f = fluids["six_probes"]
    steps_done = f.step_count
    h = {name: f.load_history(k) for k, name in enumerate(PROBES)}
    assert all(len(v["step"]) == steps_done for v in h.values())
    del fluids["no_probes"]
    kernels = {"six_probes": kernel_ms_per_step(f)}
    for name, probe in PROBES.items():
        f.set_load_probes([probe])
        kernels[name] = kernel_ms_per_step(f)
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": f.num_particles,
        "steps_per_round": args.steps,
        "steps_per_s": rates,
        "particles_identical_after_all_rounds": bool(same),
        "probe_kernels_ms_per_step": kernels,
        "last_record": {name: {"step": int(v["step"][-1]), "wetted_faces": int(v["wetted_faces"][-1]), "force": v["force"][-1].tolist()}
                        for name, v in h.items()},
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
