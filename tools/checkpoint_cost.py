"""What a checkpoint costs on the GPU: steps a scene, then times blocking saves of its state (blub_fluid_save_state: synchronise, write
path.tmp, fsync, rename) and loads of that file into a new fluid (blub_fluid_load_state, creating the fluid included).

    python tools/checkpoint_cost.py [--workload dam_256] [--steps 110] [--repeat 2] [--dir DIR]

The file goes to a temporary directory (or DIR) and is deleted afterwards.  Prints one JSON line that carries the card's name and power
limit, read in the same run.  The times are host wall clock and include the disk the file lives on; a load right after a save may be
served from the page cache.  `ms_per_step` (CUDA events over the 20 steps before the first save) puts the cost in steps.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import blub_b200  # noqa: E402
from blub_b200 import fluid as F  # noqa: E402


def card(device):
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(device)], capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="dam_256", help="scene under tests/golden/scenes")
    ap.add_argument("--steps", type=int, default=110, help="steps before the first save (the last 20 of them are timed)")
    ap.add_argument("--repeat", type=int, default=2, help="save / load pairs")
    ap.add_argument("--dir", default=None, help="directory for the state file (default: a temporary directory)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    if args.steps < 20 or args.repeat < 1:
        raise SystemExit("--steps must be at least 20 and --repeat at least 1")

    fluid = blub_b200.HybridFluid.from_scene(os.path.join(ROOT, "tests", "golden", "scenes", args.workload + ".json"), device=args.device)
    for _ in range(args.steps - 20):
        fluid.step(F.DT_120HZ)
    ms_per_step = fluid.time_steps(F.DT_120HZ, 20) / 20
    runs = []
    with tempfile.TemporaryDirectory(prefix="blub_checkpoint_", dir=args.dir) as d:
        path = os.path.join(d, "state.blub")
        for _ in range(args.repeat):
            t0 = time.perf_counter()
            fluid.save_state(path)
            t_save = time.perf_counter() - t0
            size = os.path.getsize(path)
            t0 = time.perf_counter()
            loaded = blub_b200.HybridFluid.from_state(path, device=args.device)
            t_load = time.perf_counter() - t0
            loaded.close()
            runs.append({"save_s": round(t_save, 3), "load_s": round(t_load, 3), "file_bytes": size, "save_GBps": round(size / t_save / 1e9, 3),
                         "load_GBps": round(size / t_load / 1e9, 3)})
    print(json.dumps({"workload": args.workload, "particles": fluid.num_particles, "grid": list(fluid.grid_dimension()), "at_step": fluid.step_count,
                      "ms_per_step": round(ms_per_step, 4), "runs": runs, "card": card(args.device),
                      "note": "host wall clock, including the disk of the state file's directory; the load reads the file just written (possibly "
                              "from the page cache) and includes creating the fluid"}), flush=True)
    fluid.close()


if __name__ == "__main__":
    main()
