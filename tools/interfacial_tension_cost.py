"""What interfacial tension costs on dam_256 (256^3 grid, 16.4 M particles) with half the liquid in phase B (the particles of x < 128 painted
with tag 1) at s_AB = 200 cells^3/s^2: steps/s without and with it, 3 x 60 steps each on the same step range, alternating in one process (the
order alternates too); in a run of its own under torch.profiler (eager steps) the device time per step of the new passes -- the stage-1 splat
of all particles (the density scatter's time with the tension minus without), the phase-B splat and the four interface kernels plus the
smoothing -- against the stage-9 scatter; and, when --parent DIR names a built copy of the parent commit, bench.py's default line at 0 (this
tree) alternated with the parent's, --rounds times, with its --dump-outputs arrays compared.  Reads the card name and power limit in the same
run.  Run from the repository root after python -m blub_b200.build:

    python tools/interfacial_tension_cost.py [--out profiles/h100_interfacial_tension.json] [--parent DIR] [--rounds 2]
"""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
import time

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import blub_b200  # noqa: E402
from tests import util  # noqa: E402

DT = util.DT
SIGMA = 200.0
KERNELS = ("phase_scatter_kernel", "interface_wall_kernel", "surface_smooth_kernel", "interface_curvature_kernel", "interface_rhs_kernel",
           "interface_faces_kernel")
SCATTER = "density_scatter_kernel"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def fresh(sigma):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    nx, ny, nz = f.grid_dimension()
    f.paint_tags((0, 0, 0), (nx / 2, ny, nz), 1)
    f.set_interfacial_tension(sigma, [1] if sigma else [])
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
    per = {k: 0.0 for k in KERNELS + (SCATTER, "memset", "all")}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per["all"] += e.device_time_total
        for k in KERNELS + (SCATTER,):
            if k in e.name:
                per[k] += e.device_time_total
        if "emset" in e.name:
            per["memset"] += e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in per.items()}


def steps_per_second(rounds=3, steps=60, warm=30):
    out = {0.0: [], SIGMA: []}
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
    return {"sigma_0": out[0.0], f"sigma_{SIGMA:g}_half_in_b": out[SIGMA]}


def bench_line(tree, dump):
    res = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--no-cpu-baseline", "--no-roofline", "--no-sharded-pcg", "--no-scaling-reference",
                          "--no-phases", "--dump-outputs", dump], cwd=tree, capture_output=True, text=True, timeout=1800)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        return {"error": (res.stdout + res.stderr)[-2000:]}
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_interfacial_tension.json"))
    ap.add_argument("--parent", default=None, help="a built copy of the parent commit: bench.py alternated with it")
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    result = {"card": card(), "workload": "dam_256, the particles of x < 128 in phase B", "interfacial_tension_cells3_per_s2": SIGMA}
    result["steps_per_second"] = steps_per_second()
    print(json.dumps(result["steps_per_second"]), flush=True)
    on, off = device_ms(SIGMA), device_ms(0.0)
    result["device_ms_per_step"] = {"with_interfacial_tension": on, "without": off,
                                    "stage_1_splat_of_all_particles": round(on[SCATTER] - off[SCATTER], 4),
                                    "stage_9_scatter": off[SCATTER],
                                    "phase_scatter": on["phase_scatter_kernel"],
                                    "interface_kernels_and_smoothing": round(sum(on[k] for k in KERNELS[1:]), 4),
                                    "memsets_added": round(on["memset"] - off["memset"], 4),
                                    "all_added": round(on["all"] - off["all"], 4)}
    print(json.dumps(result["device_ms_per_step"], indent=1), flush=True)
    if a.parent:
        lines = []
        with tempfile.TemporaryDirectory() as tmp:
            for r in range(a.rounds):
                for name, tree in ((("parent", a.parent), ("this", ROOT)) if r % 2 == 0 else (("this", ROOT), ("parent", a.parent))):
                    line = bench_line(tree, os.path.join(tmp, f"{name}{r}"))
                    lines.append({"round": r, "tree": name, "steps_per_s": line.get("steps_per_s", line.get("value")), "line": line})
                    print(name, lines[-1]["steps_per_s"], flush=True)
            ours, theirs = os.path.join(tmp, "this0"), os.path.join(tmp, "parent0")
            names = sorted(os.listdir(theirs)) if os.path.isdir(theirs) else []
            same = names == sorted(os.listdir(ours)) if os.path.isdir(ours) else False
            result["dump_outputs"] = {"files": len(names), "byte_identical": bool(same and names and all(
                filecmp.cmp(os.path.join(ours, n), os.path.join(theirs, n), shallow=False) for n in names))}
        result["bench_default_line_alternated"] = lines
    result["card_after"] = card()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "bench_default_line_alternated"}, indent=1))


if __name__ == "__main__":
    main()
