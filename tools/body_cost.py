"""What floating bodies cost on dam_256 (256^3 grid, 16.4 M particles): steps/s of a fluid without bodies and of one with four (two boxes, two
spheres, relative densities 0.5 to 2), 3 x 100 steps each, alternating in one process (which fluid goes first alternates too); and, in a run of
their own under torch.profiler, the device time per step of the body kernels and of the per-step copy of the borrowed solid volume into the
composite one (a 256^3 RGBA16F volume: 134 MB read and 134 MB written), next to the same copy names in a fluid without bodies.  Reads the
card name and power limit in the same run.  Run from the repository root after python -m blub_b200.build:

    python tools/body_cost.py [--out profiles/h100_bodies.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from tests import body_ref, util  # noqa: E402

DT = util.DT
BODIES = [body_ref.body("box", (12, 8, 10), 0.5, (64, 120, 64)), body_ref.body("box", (6, 6, 16), 2.0, (190, 60, 190), (0.9659258, 0.0, 0.2588190, 0.0)),
          body_ref.body("sphere", 10, 0.8, (128, 90, 200)), body_ref.body("sphere", 14, 1.2, (200, 150, 60))]
NAMES = ("body_composite_kernel", "body_load_kernel", "body_integrate_kernel", "Memcpy", "Memset")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def device_ms_per_step(f, steps=10):
    """torch.profiler device time per step of the body kernels and of all copies / memsets, over `steps` eagerly launched steps (the profiler
    does not list the copy nodes of a replayed graph) with a borrowed solid volume set, so that the composite volume is a device copy."""
    f.set_graph_replay(False)
    f.step(DT)
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(steps):
            f.step(DT)
        f.synchronize()
    per = {k: 0.0 for k in NAMES}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k in NAMES:
                if k in e.name:
                    per[k] += e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_bodies.json"))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    fluids = {"no_bodies": blub_b200.HybridFluid.from_scene(scene), "four_bodies": blub_b200.HybridFluid.from_scene(scene)}
    fluids["four_bodies"].set_bodies(BODIES)
    for f in fluids.values():
        f.step(DT)  # step 0 (rebinning) and the graph captures
        f.time_steps(DT, 9)
    rates = {k: [] for k in fluids}
    for r in range(args.rounds):
        for name, f in (list(fluids.items()) if r % 2 == 0 else list(fluids.items())[::-1]):
            rates[name].append(round(args.steps / (f.time_steps(DT, args.steps) / 1000.0), 2))
    f = fluids["four_bodies"]
    h = [f.body_history(i) for i in range(len(BODIES))]
    assert all(len(v["step"]) == f.step_count for v in h)
    dims = f.grid_dimension()
    borrowed = torch.zeros((dims[2], dims[1], dims[0], 4), dtype=torch.float16, device="cuda:0")
    torch.cuda.synchronize()
    for g in fluids.values():
        g.set_solid_voxels(borrowed.data_ptr())
    kernels = {name: device_ms_per_step(g) for name, g in fluids.items()}
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": f.num_particles,
        "bodies": BODIES,
        "steps_per_round": args.steps,
        "steps_per_s": rates,
        "device_ms_per_step": kernels,
        "composite_copy_bytes": 2 * 256 ** 3 * 8,
        "last_pose": [{"step": int(v["step"][-1]), "centre": v["centre"][-1].tolist(), "velocity": v["velocity"][-1].tolist(),
                       "wetted_faces": int(v["wetted_faces"][-1])} for v in h],
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
