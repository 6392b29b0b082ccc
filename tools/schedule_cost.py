"""What the density scatter's brick schedule costs and gives on the 256^3 dam break: stage times of eagerly launched steps (CUDA events around
every stage, HybridFluid.step_timed) over one sort window, with the schedule and with BLUB_SCATTER_SCHEDULE=off, each mode in a fresh process.
Stage 3 of a re-sort step holds the binning and, with the schedule, its build; stage 9 is the density scatter with its rhs.

    python tools/schedule_cost.py [--first 224] [--steps 9] [--out FILE.json]

Needs a GPU; fails without one.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def measure(first, steps):
    sys.path.insert(0, ROOT)
    import blub_b200
    from blub_b200 import fluid as F

    f = blub_b200.HybridFluid.from_scene(os.path.join(ROOT, "tests", "golden", "scenes", "dam_256.json"))
    for _ in range(first):
        f.step(F.DT_120HZ)
    f.synchronize()
    rows = []
    for k in range(first, first + steps):
        ms = f.step_timed(F.DT_120HZ)
        rows.append({"step": k, "resort": k % 8 == 0, "stage_ms": {n: round(v, 4) for n, v in zip(F.STAGES, ms)}, "total_ms": round(sum(ms), 4)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--first", type=int, default=224)
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(measure(a.first, a.steps)))
        return
    result = {}
    for mode in ("schedule", "off"):
        env = dict(os.environ)
        env.pop("BLUB_SCATTER_SCHEDULE", None)
        if mode == "off":
            env["BLUB_SCATTER_SCHEDULE"] = "off"
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--first", str(a.first), "--steps", str(a.steps)], env=env,
                           capture_output=True, text=True, check=True)
        result[mode] = json.loads(r.stdout.strip().splitlines()[-1])
    text = json.dumps(result, indent=1)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
