"""What particle tags cost on dam_256 (16.4 M particles): steps/s of an untagged fluid and of a fluid tagged with index tags (tag = particle
index), 3 x 100 steps each, alternating in one process (which fluid goes first alternates too); and the time of one tag census (CUDA events around repeated calls on the fluid's
stream, which include the two small copies of the census records and the host synchronisation; torch.profiler for the kernel alone), with
256 tags and with 1 tag.  Reads the card name and power limit in the same run.  Run from the repository root after python -m blub_b200.build:

    python tools/tag_cost.py [--out profiles/h100_tags.json]
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
from tests.test_gpu_tags import set_tags  # noqa: E402

DT = util.DT


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def census_ms(f, first, count, calls=20):
    """(ms per call with CUDA events on the fluid's stream, ms of tag_census_kernel per call with torch.profiler)"""
    stream = torch.cuda.ExternalStream(f.stream())
    f.tag_census(first, count)  # warm
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(calls):
        f.tag_census(first, count)
    e1.record(stream)
    e1.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(calls):
            f.tag_census(first, count)
    kernel = sum(e.device_time_total for e in p.events() if "tag_census_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA)
    return round(e0.elapsed_time(e1) / calls, 4), round(kernel / calls / 1000, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_tags.json"))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    fluids = {"untagged": blub_b200.HybridFluid.from_scene(scene), "index_tags": blub_b200.HybridFluid.from_scene(scene)}
    n = fluids["index_tags"].num_particles
    set_tags(fluids["index_tags"], np.arange(n, dtype=np.uint32))
    set_tags(fluids["untagged"], np.zeros(n, dtype=np.uint32))  # the same upload on both fluids
    for f in fluids.values():
        f.step(DT)  # step 0 (rebinning) and the graph captures
        f.time_steps(DT, 9)
    rates = {k: [] for k in fluids}
    for r in range(args.rounds):  # the same step range for both fluids; which one goes first alternates
        for name, f in (list(fluids.items()) if r % 2 == 0 else list(fluids.items())[::-1]):
            rates[name].append(round(args.steps / (f.time_steps(DT, args.steps) / 1000.0), 2))
    for f in fluids.values():
        f.synchronize()
    same = np.array_equal(fluids["untagged"].download_particles()[:, :3], fluids["index_tags"].download_particles()[:, :3])
    assert np.array_equal(np.sort(fluids["index_tags"].particle_tags()), np.arange(n, dtype=np.uint32))
    f = fluids["index_tags"]
    del fluids["untagged"]
    census = {"index_tags_256": census_ms(f, 0, 256)}  # 256 particles in range: positions only are read for the rest
    set_tags(f, (np.arange(n, dtype=np.uint32) // 1000) % 256)  # every particle in range, runs of 1000 after the binning order
    census["all_in_range_256"] = census_ms(f, 0, 256)
    census["all_in_range_1"] = census_ms(f, 0, 1)
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": n,
        "steps_per_round": args.steps,
        "steps_per_s": rates,
        "positions_identical_after_all_rounds": bool(same),
        "census_ms": {k: {"call_events": v[0], "kernel_profiler": v[1]} for k, v in census.items()},
        "census_bytes_read_all_in_range": n * 64,
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
