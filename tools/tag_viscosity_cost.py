"""What a tag viscosity table costs on dam_256: steps/s over steps 30-90 of four fluids stepped alternately in one process (no viscosity,
uniform nu at k = nu dt = 1, half the liquid tagged at k = 1 and the rest nu = 0, a uniform table at k = 1), with the stage-0 time and the
solve iterations; then, in a run of its own under torch.profiler (eager steps), the device time per step of the cell, set-up and solve kernels
of the half-tagged and the uniform-nu fluids.  Reads the card name and power limit in the same run.  Run from the repository root after
python -m blub_b200.build:

    python tools/tag_viscosity_cost.py [--out profiles/h100_tag_viscosity.json]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blub_b200  # noqa: E402
from tests import util  # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from viscosity_cost import card  # noqa: E402

DT = util.DT
NAMES = ("tag_density_scatter_kernel", "tag_viscosity_finish_kernel", "viscosity_setup_kernel", "viscosity_list_kernel", "viscosity_solve_kernel")
# per live face and iteration, counted from viscosity_kernels.cu: the constant solve's 88 B (tools/viscosity_cost.py), plus, in each of the two
# row evaluations (s . A s and the update), the own coefficients (16 B, of which the diagonal is also read by z = r / diagonal) and up to
# three -d coefficients from the neighbours (3 x 4 B), and the diagonal again in the new-direction pass (4 B)
BYTES_PER_FACE_ITERATION_CONSTANT = (7 + 11 + 3) * 4 + 3 * 4 / 3
BYTES_PER_FACE_ITERATION_PAIRS = BYTES_PER_FACE_ITERATION_CONSTANT + 2 * (16 + 3 * 4) + 4


def make(kind, dt32):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    nu = 1.0 / dt32
    if kind == "uniform_nu":
        f.set_viscosity(nu)
    elif kind == "half_tagged":
        nx, ny, nz = f.grid_dimension()
        f.paint_tags((0, 0, 0), (nx // 2, ny, nz), 1)
        f.set_tag_viscosities({1: nu})
    elif kind == "uniform_table":
        f.set_viscosity(nu)
        f.set_tag_viscosities({0: nu})
    return f


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
    it = sum(iterations) / steps
    return {"device_ms_per_step": ms, "iterations_per_solve": it,
            "solve_us_per_iteration": round(1000 * ms["viscosity_solve_kernel"] / max(it, 1e-9), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_tag_viscosity.json"))
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dt32 = float(np.float32(DT))
    kinds = ("none", "uniform_nu", "half_tagged", "uniform_table")
    fluids = {k: make(k, dt32) for k in kinds}
    for f in fluids.values():
        f.step(DT)
        f.time_steps(DT, 29)  # to step 30
    rates, stage0, iterations = {k: [] for k in kinds}, {k: [] for k in kinds}, {k: [] for k in kinds}
    window = 60 // args.rounds  # steps 30-90 in rounds, the order alternating
    for r in range(args.rounds):
        for name in (kinds if r % 2 == 0 else kinds[::-1]):
            f = fluids[name]
            rates[name].append(round(window / (f.time_steps(DT, window) / 1000.0), 2))
    for name, f in fluids.items():
        for _ in range(5):
            stage0[name].append(f.step_timed(DT)[0])
            iterations[name].append(f.last_viscosity_solve()[0] if name != "none" else 0)
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": fluids["none"].num_particles,
        "k": 1.0,
        "steps_per_s_30_90": rates,
        "stage0_ms_median_steps_91_95": {k: round(statistics.median(v), 3) for k, v in stage0.items()},
        "iterations_per_solve_steps_91_95": {k: v for k, v in iterations.items()},
        "bytes_per_face_iteration": {"constant": BYTES_PER_FACE_ITERATION_CONSTANT, "pairs": BYTES_PER_FACE_ITERATION_PAIRS},
    }
    for name in ("uniform_nu", "half_tagged", "uniform_table"):
        out[f"profile_{name}"] = profile_steps(fluids[name])
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
