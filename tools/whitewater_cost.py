"""What whitewater costs on dam_256 (256^3 grid, 16.4 M particles): the step time with and without it over steps 200-230, alternating in one
process in rounds of 10 steps (graph replay; the order alternates too), and then, under torch.profiler with eager steps, the device time per
step of the whitewater kernels and of all kernels over steps 230-240 of both fluids.  The whitewater fluid runs the default setting
(blub_b200.fluid.WHITEWATER_DEFAULTS) with room for 4 M particles from step 0; the liquid is the same in both.  Reads the card name and power
limit in the same run.  Run from the repository root after python -m blub_b200.build:

    python tools/whitewater_cost.py [--out profiles/h100_whitewater.json]
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
CAPACITY = 4 << 20
KERNELS = ("whitewater_update_kernel", "whitewater_compact_kernel", "whitewater_potential_kernel", "whitewater_emit_kernel")
SCANS = ("scan_block_sums_kernel", "scan_sums_kernel", "scan_apply_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def device_ms(f, steps=10):
    f.set_graph_replay(False)
    f.step(DT)  # the eager launches' first use
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(steps):
            f.step(DT)
        f.synchronize()
    per = {k: 0.0 for k in KERNELS + SCANS + ("all",)}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per["all"] += e.device_time_total
        for k in KERNELS + SCANS:
            if k in e.name:
                per[k] += e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_whitewater.json"))
    a = ap.parse_args()
    result = {"card": card(), "workload": "dam_256, whitewater with the default setting and a capacity of 4 M from step 0", "capacity": CAPACITY}
    fluids = {"without": blub_b200.HybridFluid.from_scene(util.scene_path("dam_256")),
              "with_whitewater": blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))}
    fluids["with_whitewater"].set_whitewater(CAPACITY)
    for f in fluids.values():
        for _ in range(200):
            f.step(DT)
        f.synchronize()
    ms = {k: [] for k in fluids}
    for r in range(3):  # steps 200-230 in rounds of 10
        for name in (list(fluids) if r % 2 == 0 else list(fluids)[::-1]):
            f = fluids[name]
            f.synchronize()
            t0 = time.perf_counter()
            for _ in range(10):
                f.step(DT)
            f.synchronize()
            ms[name].append(round((time.perf_counter() - t0) / 10 * 1000, 4))
    result["ms_per_step_steps_200_230"] = ms
    result["whitewater_counters_at_230"] = fluids["with_whitewater"].whitewater_counters
    print(json.dumps(result, indent=1), flush=True)
    on, off = device_ms(fluids["with_whitewater"]), device_ms(fluids["without"])
    result["device_ms_per_step_steps_231_240"] = {"with_whitewater": on, "without": off,
                                                  "whitewater_kernels": round(sum(on[k] for k in KERNELS), 4),
                                                  "scans_added": round(sum(on[k] - off[k] for k in SCANS), 4),
                                                  "all_added": round(on["all"] - off["all"], 4)}
    result["whitewater_counters_at_241"] = fluids["with_whitewater"].whitewater_counters
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
