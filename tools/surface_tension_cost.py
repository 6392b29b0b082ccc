"""What surface tension costs on dam_256 (256^3 grid, 16.4 M particles) at water's value for 1 cm cells (72.8 cells^3/s^2): steps/s without and
with it, 3 x 100 steps each on the same step range, alternating in one process (the order alternates too); in a run of its own under
torch.profiler (eager steps) the device time per step of the new passes -- the stage-1 splat (the density scatter's time per step with surface
tension minus without) and the four surface kernels -- against the stage-9 scatter; and, when --parent DIR names a built copy of the parent
commit, bench.py's default line at 0 (this tree) alternated with the parent's, --rounds times.  Reads the card name and power limit in the same
run.  Run from the repository root after python -m blub_b200.build:

    python tools/surface_tension_cost.py [--out profiles/h100_surface_tension.json] [--parent DIR] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import blub_b200  # noqa: E402
from tests import util  # noqa: E402

DT = util.DT
WATER_1CM = 7.28e-5 / (0.01 ** 3)
SURFACE = ("surface_wall_kernel", "surface_smooth_kernel", "surface_curvature_kernel", "surface_rhs_kernel", "surface_faces_kernel")
SCATTER = "density_scatter_kernel"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def fresh(sigma):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    f.set_surface_tension(sigma)
    return f


def device_ms(sigma, warm=40, steps=10):
    f = fresh(sigma)
    for _ in range(warm):
        f.step(DT)
    f.set_graph_replay(False)
    f.step(DT)
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(steps):
            f.step(DT)
        f.synchronize()
    per = {k: 0.0 for k in SURFACE + (SCATTER, "memset", "all")}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per["all"] += e.device_time_total
        for k in SURFACE + (SCATTER,):
            if k in e.name:
                per[k] += e.device_time_total
        if "emset" in e.name:
            per["memset"] += e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in per.items()}


def steps_per_second(rounds=3, steps=100, warm=30):
    out = {0.0: [], WATER_1CM: []}
    fluids = {s: fresh(s) for s in out}
    for f in fluids.values():
        for _ in range(warm):
            f.step(DT)
        f.synchronize()
    for r in range(rounds):
        order = list(out) if r % 2 == 0 else list(out)[::-1]
        for s in order:
            f = fluids[s]
            f.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                f.step(DT)
            f.synchronize()
            out[s].append(round(steps / (time.perf_counter() - t0), 2))
    return {"sigma_0": out[0.0], "sigma_water_1cm": out[WATER_1CM]}


def bench_line(tree):
    res = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--no-cpu-baseline", "--no-roofline", "--no-sharded-pcg", "--no-scaling-reference",
                          "--no-phases"], cwd=tree, capture_output=True, text=True, timeout=1800)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        return {"error": (res.stdout + res.stderr)[-2000:]}
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_surface_tension.json"))
    ap.add_argument("--parent", default=None, help="a built copy of the parent commit: bench.py alternated with it")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    result = {"card": card(), "workload": "dam_256", "surface_tension_cells3_per_s2": WATER_1CM}
    result["steps_per_second"] = steps_per_second()
    on, off = device_ms(WATER_1CM), device_ms(0.0)
    result["device_ms_per_step"] = {"with_surface_tension": on, "without": off,
                                    "stage_1_splat": round(on[SCATTER] - off[SCATTER], 4),
                                    "stage_9_scatter": off[SCATTER],
                                    "surface_kernels": round(sum(on[k] for k in SURFACE), 4),
                                    "memsets_added": round(on["memset"] - off["memset"], 4)}
    print(json.dumps(result["device_ms_per_step"], indent=1), flush=True)
    if a.parent:
        lines = []
        for r in range(a.rounds):
            for name, tree in ((("parent", a.parent), ("this", ROOT)) if r % 2 == 0 else (("this", ROOT), ("parent", a.parent))):
                line = bench_line(tree)
                lines.append({"round": r, "tree": name, "steps_per_s": line.get("steps_per_s", line.get("value")), "line": line})
                print(name, lines[-1]["steps_per_s"], flush=True)
        result["bench_default_line_alternated"] = lines
    result["card_after"] = card()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
