"""What a moving tank costs on dam_256 (256^3 grid, 16.4 M particles).  Run from the repository root after python -m blub_b200.build:

    python tools/tank_cost.py [--out profiles/h100_tank.json] [--rounds 3] [--steps 60]

  steps/s    dam_256 from the scene, the same step range [30, 30 + steps) with no frame, a translating frame (a surge harmonic) and a rolling
             frame (the surge plus a roll about z through the tank's centre), a new frame before every step; the three in alternating rounds,
             device time from CUDA events around the timed steps
  kernel     tank_frame_kernel's device time from CUDA events around 100 launches of stage 0 with and without the rolling frame at step 30 (the
             difference per launch), and from torch.profiler; its bytes (112 per particle) over that time against the 3.35 TB/s of the H100 SXM
             data sheet
Reads the card name and power limit in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from blub_b200 import fluid as F  # noqa: E402
from tests import util  # noqa: E402

BYTES_PER_PARTICLE = 112  # 3 velocity rows read and written, the position read: 7 float4
HBM_TB_S = 3.35
DT = F.DT_120HZ
SURGE = {"pivot": (128.0, 64.0, 128.0), "translations": [{"direction": (1.0, 0.0, 0.0), "amplitude": 8.0, "frequency": 0.5, "phase": 0.0}]}
ROLL = dict(SURGE, rotation={"axis": (0.0, 0.0, 1.0), "amplitude": 0.1, "frequency": 0.4, "phase": 0.0, "rate": 0.0})
MOTIONS = {"none": None, "translating": SURGE, "rolling": ROLL}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def advance_to(f, motion, first):
    for k in range(first):
        if motion is not None:
            f.set_tank_frame(F.tank_frame_at(motion, k * DT))
        f.step(DT)
    f.synchronize()


def timed_steps(scene, motion, first, steps):
    f = blub_b200.HybridFluid.from_scene(scene)
    advance_to(f, motion, first)
    stream = torch.cuda.ExternalStream(f.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for k in range(first, first + steps):
        if motion is not None:
            f.set_tank_frame(F.tank_frame_at(motion, k * DT))
        f.step(DT)
    e1.record(stream)
    e1.synchronize()
    return steps / (e0.elapsed_time(e1) / 1000.0)


def stage0_ms(f, launches):
    stream = torch.cuda.ExternalStream(f.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(launches):
        f.step_stages(DT, 0, 1)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / launches


def kernel_time(scene, first=30, launches=100):
    f = blub_b200.HybridFluid.from_scene(scene)
    f.set_graph_replay(False)
    advance_to(f, ROLL, first)
    n = f.num_particles
    frame = F.tank_frame_at(ROLL, first * DT)
    # stage 0 re-run in place: the P2G rewrites the grid from the same particles, the frame kernel turns the rows a little further each time
    ms = {}
    for rnd in range(3):
        for name in ("rolling", "none"):
            f.set_tank_frame(frame if name == "rolling" else None)
            stage0_ms(f, 5)
            ms.setdefault(name, []).append(stage0_ms(f, launches))
            f.step_stages(DT, 1, 14)  # the rest of the step, so that the next frame can be set
    f.set_tank_frame(frame)
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(launches):
            f.step_stages(DT, 0, 1)
    f.step_stages(DT, 1, 14)
    f.synchronize()
    times = [e.device_time_total for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "tank_frame_kernel" in e.name]
    diff = [a - b for a, b in zip(ms["rolling"], ms["none"])]
    us = statistics.median(times) if times else float("nan")
    return {"particles": n, "bytes": n * BYTES_PER_PARTICLE, "stage0_ms_rolling": [round(x, 4) for x in ms["rolling"]],
            "stage0_ms_none": [round(x, 4) for x in ms["none"]], "event_difference_ms": [round(x, 4) for x in diff],
            "profiler_launches": len(times), "kernel_us_median": round(us, 2), "kernel_us_min": round(min(times), 2) if times else None,
            "kernel_us_max": round(max(times), 2) if times else None,
            "tb_per_s": round(n * BYTES_PER_PARTICLE / (us * 1e-6) / 1e12, 3),
            "share_of_3_35_tb_s": round(n * BYTES_PER_PARTICLE / (us * 1e-6) / 1e12 / HBM_TB_S, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_tank.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--first", type=int, default=30)
    ap.add_argument("--steps", type=int, default=60)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    out = {"card": card(), "workload": "dam_256", "dt": DT, "step_range": [args.first, args.first + args.steps], "motions": MOTIONS}
    rates = {name: [] for name in MOTIONS}
    for _ in range(args.rounds):
        for name, motion in MOTIONS.items():
            rates[name].append(round(timed_steps(scene, motion, args.first, args.steps), 2))
            print(name, rates[name][-1], flush=True)
    out["steps_per_s"] = rates
    out["kernel"] = kernel_time(scene, args.first)
    print(json.dumps(out["kernel"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
