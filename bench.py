#!/usr/bin/env python
"""bench.py -- steps/sec of the blub fluid step on H100 + PCG roofline + CPU baseline (contract: see DESIGN.md section 6).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl blub|reference] [--workload dam_256] [--multi sharded|replicas]
                    [--dump-outputs DIR]

A "step" is one HybridFluid::step (P2G, PCG solve, G2P/advection, density rhs, PCG solve, particle correction) over the
synthetic 256^3 / 16,387,064-particle dam break that BASELINE.json's metric is quoted on.  N > 1 (torchrun, one rank per
GPU): ONE simulation on a 256 x 256 x 256N grid sharded into N z-slabs (weak scaling: per-GPU work fixed -- a z-uniform dam
with the same 16.3 M particles per slab); `value` = slab-steps/s = N * steps/s.  The N = 1 line carries `scaling_reference`, the
same per-slab scene on one GPU.  `--multi stacked` stacks N dam_256 cubes instead, `--multi replicas` runs N independent scenes.
`--impl reference`: the reference (Rust + wgpu/Vulkan) cannot run on this image, so this arm times the CPU restatement of
its algorithm (oracle/) on the host cores -- the only place besides cpu_baseline where bench.py executes oracle/.
`--dump-outputs DIR`: after the K timed steps, the state the timed path left (the ten arrays of blub_fluid_view) is written to
DIR/<name>.npy (float32; fixed, seeded samples of arrays larger than a cap, <= 64 MB in all, N > 1: DIR/<name>_rank<k>.npy sharing
that budget), so that two builds can be compared.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "simulation steps/sec"
SCENES = os.path.join(ROOT, "tests", "golden", "scenes")


def scene_path(name):
    return os.path.join(SCENES, name + ".json")


# Workloads that carry a moving solid (SURVEY section 8d, config C5): the scene's fluid + an analytic box written into the solid-voxel
# volume before every step, as Scene::step does with its meshes (src/scene/mod.rs:192-211).  Box of 24x40x24 cells travelling +-20 cells
# about the middle of the basin, SmoothStep over 2 s (animation parameters of scenes/#double_dam_wgpulogo_rotating.json:61-79).
SOLID_WORKLOADS = {
    "double_dam_box": {"scene": "double_dam",
                       "solid": {"world_position": [0.44, 0.20, 0.32], "scale": 1.0, "rotation_angles": [0.0, 0.0, 0.0], "shape": "box",
                                 "half_extent": [0.12, 0.20, 0.12], "translation": {"target": [0.84, 0.20, 0.32], "curve": "SmoothStep", "duration": 2.0}}},
}


def workload_scene(name):
    return SOLID_WORKLOADS[name]["scene"] if name in SOLID_WORKLOADS else name


def workload_desc(name):
    sc = json.load(open(scene_path(workload_scene(name))))
    d = sc["fluid"]["grid_dimension"]
    extra = " + moving solid box (voxelized every step)" if name in SOLID_WORKLOADS else ""
    return sc, f"{name}: {d['x']}x{d['y']}x{d['z']} grid{extra}"


class SolidStepper:
    """Scene::step for a workload with a solid: advance the clock, voxelize on the fluid's stream, step the fluid."""

    def __init__(self, fluid, sc, solid, device):
        import torch
        d = sc["fluid"]["grid_dimension"]
        self.fluid, self.solid, self.dims = fluid, solid, (d["x"], d["y"], d["z"])
        self.scale = sc["fluid"]["grid_to_world_scale"]
        self.origin = [sc["fluid"]["world_position"][c] for c in "xyz"]
        self.vol = torch.zeros((d["z"], d["y"], d["x"], 4), dtype=torch.float16, device=f"cuda:{device}")
        torch.cuda.synchronize()
        fluid.set_solid_voxels(self.vol.data_ptr())
        self.stream = torch.cuda.ExternalStream(fluid.stream(), device=f"cuda:{device}")
        self.t = 0.0

    def step(self, dt):
        from blub_b200 import fluid as F
        self.t += dt
        F.solid_voxelize(self.vol.data_ptr(), self.dims, self.solid, self.scale, self.origin, self.t, dt, cuda_stream=self.fluid.stream())
        self.fluid.step(dt)

    def time_steps(self, dt, steps):
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        for _ in range(steps):
            self.step(dt)
        e1.record(self.stream)
        e1.synchronize()
        return float(e0.elapsed_time(e1))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""

    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", str(self.index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.12)
        self.proc.terminate()
        sm = sorted(int(r[0]) for r in self.rows if r and r[0].isdigit())
        mx = [int(r[1]) for r in self.rows if len(r) > 1 and r[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for k, n in enumerate(names) if any(len(r) > 2 + k and r[2 + k].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons, "samples": len(sm)}


DUMP_PARTICLES = 1 << 18  # particles sampled per particle array (4 floats each)
DUMP_CELLS = 1 << 20      # cells sampled per grid volume


def _sample(n, cap, seed):
    """All indices when n <= cap, else `cap` distinct indices drawn with a fixed seed, ascending."""
    import numpy as np

    if n <= cap:
        return np.arange(n, dtype=np.int64)
    return np.sort(np.random.default_rng(seed).choice(n, size=cap, replace=False))


def dump_outputs(fluid, out_dir, suffix="", parts=1):
    """The ten arrays a renderer binds after a step (blub_fluid_view), as float32 .npy files.  Particle arrays are (n, 4) in
    the library's particle order; grid volumes are flattened in x-fastest order.  Arrays above the caps are sampled at indices
    drawn with a fixed seed, stored beside them in float64 (particle_index, cell_index).  At most ~50 MB in all: with `parts`
    ranks dumping into the same directory each one gets 1/parts of the caps."""
    import numpy as np

    from blub_b200 import fluid as F

    os.makedirs(out_dir, exist_ok=True)
    fluid.synchronize()
    n = fluid.num_particles
    pi = _sample(n, DUMP_PARTICLES // parts, 1)
    files = {"particle_index": pi.astype(np.float64)}
    for name, tap in (("particles_position", F.TAP_POS), ("particles_velocity_x", F.TAP_VX), ("particles_velocity_y", F.TAP_VY),
                      ("particles_velocity_z", F.TAP_VZ)):
        files[name] = fluid.download_particles(tap)[pi]
    ci = _sample(fluid.n, DUMP_CELLS // parts, 2)
    files["cell_index"] = ci.astype(np.float64)
    for name, tap in (("grid_velocity_x", F.TAP_UX), ("grid_velocity_y", F.TAP_UY), ("grid_velocity_z", F.TAP_UZ), ("marker", F.TAP_MARKER),
                      ("pressure_from_velocity", F.TAP_P_VEL), ("pressure_from_density", F.TAP_P_DEN)):
        files[name] = fluid.download_grid(tap).reshape(-1)[ci].astype(np.float32)
    for name, a in files.items():
        np.save(os.path.join(out_dir, name + suffix + ".npy"), np.ascontiguousarray(a))
    return {"dir": out_dir, "particles": n, "particles_dumped": int(pi.size), "cells_dumped": int(ci.size),
            "bytes": int(sum(a.nbytes for a in files.values()))}


def pcg_roofline(device, n=256, reps=5):
    """SURVEY 8(d) microbench: n^3 grid, all interior cells FLUID, rhs ~ U[-1,1) (seed 1234) mean-removed, tolerance 0 so
    all 33 iterations run; algorithmic bytes = (42 * 33 + 21) * N per solve."""
    import numpy as np

    import blub_b200
    from blub_b200 import fluid as F

    f = blub_b200.HybridFluid(n, n, n, 8, device=device)
    m = np.zeros((n, n, n), dtype=np.int8)
    m[1:-1, 1:-1, 1:-1] = 1
    rng = np.random.default_rng(1234)
    b = rng.uniform(-1.0, 1.0, (n, n, n)).astype(np.float32)
    b -= b[m == 1].mean(dtype=np.float64).astype(np.float32)
    b[m != 1] = 0
    f.upload_grid(F.TAP_MARKER, m)
    f.upload_grid(F.TAP_RESIDUAL, b)
    f.set_solver_config(0, error_tolerance=0.0, max_num_iterations=32, error_check_frequency=4)
    dt = F.DT_120HZ
    f.time_solve(0, dt, 2)  # warm-up
    ms = sorted(f.time_solve(0, dt, reps))
    t = ms[len(ms) // 2] * 1e-3
    cells = n ** 3
    bytes_alg = (42 * 33 + 21) * cells
    peaks = {}
    src = "H100 SXM data sheet, 3350 GB/s"
    peak = 3350.0
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
        peak = float(peaks.get("hbm_gbs", peak))
        src = "MEASURED_PEAKS.json hbm_gbs (burst copy)"
    traffic = traffic_src = None  # DRAM bytes actually moved need a hardware profiler: not measured
    ach = bytes_alg / t / 1e9
    e, it = f.last_solve(0)
    f.close()
    return {"bound": "hbm", "achieved": round(ach, 1), "peak": peak, "unit": "GB/s", "frac": round(ach / peak, 4), "traffic": traffic,
            "kernel": "PCG solve (init + 33 x {dot, update, search})", "grid": f"{n}^3 all-fluid", "ms_per_solve": round(t * 1e3, 4),
            "algorithmic_bytes_per_solve": bytes_alg, "peak_source": src, "iterations_run": it + 1, "max_num_iterations": it, "traffic_source": traffic_src}


def pcg_sharded(rank, world, local, n=512, reps=5):
    """Strong-scaling PCG microbench: the n^3 all-fluid box cut into `world` z-slabs, one per GPU; boundary planes travel as
    P2P stores inside the persistent kernel, scalars through peer mailboxes (windows exchanged once via CUDA IPC)."""
    import numpy as np
    import torch.distributed as dist

    import blub_b200
    from blub_b200 import fluid as F

    nz_owned = n // world
    f = blub_b200.HybridFluid.create_slab(n, n, nz_owned, 8, rank=rank, world=world, device=local)
    from blub_b200 import slab

    handles = slab.exchange_handles(f.ipc_export_window(), dist)
    own = f.slab_window()[0]
    windows = [own if k == rank else F.ipc_open(handles[k], local) for k in range(world)]
    f.attach_slab_peers(windows)
    halo = 4
    z0 = rank * nz_owned - halo
    m = np.zeros((nz_owned + 2 * halo, n, n), dtype=np.int8)
    zz = np.arange(z0, z0 + nz_owned + 2 * halo)
    inside = (zz >= 1) & (zz <= n - 2)
    m[inside, 1:-1, 1:-1] = 1
    rng = np.random.default_rng(1234 + rank)
    b = rng.uniform(-1.0, 1.0, m.shape).astype(np.float32)
    b[m != 1] = 0
    b[:halo] = 0
    b[halo + nz_owned:] = 0
    f.upload_grid(F.TAP_MARKER, m)
    f.upload_grid(F.TAP_RESIDUAL, b)
    f.set_solver_config(0, error_tolerance=0.0, max_num_iterations=32, error_check_frequency=4)
    dist.barrier()
    f.time_solve(0, F.DT_120HZ, 2)
    dist.barrier()
    ms = f.time_solve(0, F.DT_120HZ, reps)
    t = torch_max(sorted(ms)[len(ms) // 2])
    e, it = f.last_solve(0)
    dist.barrier()
    f.close()
    bytes_alg = (42 * 33 + 21) * n ** 3
    return {"grid": f"{n}^3 all-fluid, {world} z-slabs of {nz_owned} planes", "ms_per_solve": round(t, 4), "iterations": it,
            "aggregate_GBps": round(bytes_alg / (t * 1e-3) / 1e9, 1), "per_gpu_GBps": round(bytes_alg / (t * 1e-3) / 1e9 / world, 1),
            "exchange": "in-kernel P2P stores + mailbox all-reduce over NVLink (no NCCL in the solve)"}


def torch_max(x):
    import torch
    import torch.distributed as dist

    t = torch.tensor([x], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def oracle_stepper(f, sc, workload):
    """One Scene::step on the oracle: with a solid workload the box is re-voxelized (NumPy restatement) before every fluid step."""
    from oracle import oracle as O

    if workload not in SOLID_WORKLOADS:
        return lambda: f.step(O.DT_120HZ)
    from oracle import solids as S

    d = sc["fluid"]["grid_dimension"]
    state = {"t": 0.0}

    def step():
        state["t"] += O.DT_120HZ
        vol, _ = S.voxelize(SOLID_WORKLOADS[workload]["solid"], (d["x"], d["y"], d["z"]), sc["fluid"]["grid_to_world_scale"],
                            [sc["fluid"]["world_position"][c] for c in "xyz"], state["t"], O.DT_120HZ)
        f.set_voxels(vol)
        f.step(O.DT_120HZ)
    return step


def cpu_baseline_sample(workload, steps):
    """Oracle (CPU port of the reference's algorithm) timed on this box's host cores on `steps` steps of the workload."""
    from oracle import oracle as O

    sc = O.load_scene(scene_path(workload_scene(workload)))
    f = O.fluid_from_scene(sc)
    step = oracle_stepper(f, sc, workload)
    step()  # first step pays page faults / first-touch; not timed
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    t = time.perf_counter() - t0
    cores = os.cpu_count() or 1
    return {"value": round(steps / t, 5), "unit": "steps/s", "cores": cores, "kind": "port",
            "sample": f"{steps} step(s) of {workload} after 1 untimed step, OpenMP over {cores} host threads (linked-list builds serial)"}


def config_block(desc, particles, dt, parallelism, window):
    """The `config` object of the JSON line -- same keys in the blub arm and in the reference arm."""
    return {"workload": desc, "particles": particles, "dt": dt, "solver": "tol 0.1 / max 32 / check 4 (reference defaults)", "rebin_every": 60,
            "parallelism": parallelism, "l2": "inputs larger than L2 (>= 1 GB of particle state, 64 MiB per grid volume)", "window": window}


def late_window_and_in_step(fluid, step, stepper, dt, steps_done, args, early_ms_per_step):
    """The timed region of the contract (K steps after W warm-up steps) is the CHEAPEST phase of a dam break: the step gets more expensive
    as the wave spreads (more active solver tiles, more surface).  So the same simulation is carried on to step `late_start` and a second
    window of 20 steps is timed there with the same method; then one eagerly launched step is timed stage by stage and the in-step PCG solves
    are put on the roofline of the bytes they TOUCH (work lists of the solver), next to the dense microbench of `roofline`."""
    import numpy as np

    from blub_b200 import fluid as F

    late_start, late_steps = args.late_start, 20
    while steps_done < late_start:
        step(dt)
        steps_done += 1
    fluid.synchronize()
    late_first = steps_done  # == late_start unless the timed regions already ran past it (large --steps): the label follows the scene, not the flag
    ms_late = stepper.time_steps(dt, late_steps) if stepper else fluid.time_steps(dt, late_steps)
    steps_done += late_steps
    phases = {"early": {"first_step": max(args.warmup, 3), "steps": args.steps, "ms_per_step": round(early_ms_per_step, 4), "steps_per_s": round(1e3 / early_ms_per_step, 3)},
              "late": {"first_step": late_first, "steps": late_steps, "ms_per_step": round(ms_late / late_steps, 4), "steps_per_s": round(late_steps / (ms_late * 1e-3), 3)}}
    if stepper:
        return phases, None, None, steps_done
    stage_ms = fluid.step_timed(dt)
    steps_done += 1
    work = fluid.solver_work()  # of the density solve (the last one); the velocity solve of the same step walks almost the same lists
    it = [fluid.last_solve(w)[1] for w in (0, 1)]
    touched_cells = work["tiles"] * work["cells_per_tile"] + work["columns"] * work["cells_per_column"]
    m = fluid.download_grid(F.TAP_MARKER)
    fluid_cells = int((m == 1).sum())
    peak = 3350.0  # H100 SXM data sheet
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk)).get("hbm_gbs", peak))
    solves = []
    for which, stage in ((0, 2), (1, 10)):
        passes = it[which] + 1  # iterations 0 .. it are run (pressure_solver.rs:654-723)
        t = stage_ms[stage] * 1e-3
        b_touched, b_fluid = (42 * passes + 21) * touched_cells, (42 * passes + 21) * fluid_cells
        solves.append({"solve": F.STAGES[stage], "ms": round(stage_ms[stage], 4), "iterations_run": passes,
                       "touched_GBps": round(b_touched / t / 1e9, 1), "touched_frac_of_hbm_peak": round(b_touched / t / 1e9 / peak, 4),
                       "fluid_cell_GBps": round(b_fluid / t / 1e9, 1), "fluid_cell_frac_of_hbm_peak": round(b_fluid / t / 1e9 / peak, 4)})
    in_step = {"at_step": steps_done - 1, "fluid_cells": fluid_cells, "fluid_fraction": round(fluid_cells / fluid.n, 4),
               "solver_work": work, "touched_cells": touched_cells, "bytes_per_cell_and_pass": 42, "solves": solves,
               "stage_ms": {name: round(v, 4) for name, v in zip(F.STAGES, stage_ms)}, "stage_total_ms": round(float(sum(stage_ms)), 4),
               "note": "touched = cells of the tiles and quad columns on the solver's work lists; the HBM roofline of the kernel is the dense microbench in `roofline`"}
    # what a consumer pays to GET the result: nothing on the device (blub_fluid_view hands out the ten device pointers the renderer binds,
    # hybrid_fluid.rs:351-369); a host copy of the particle positions is a plain D2H transfer
    t0 = time.perf_counter()
    pos = fluid.download_particles()
    t_dl = time.perf_counter() - t0
    t0 = time.perf_counter()
    fluid.view()
    t_view = time.perf_counter() - t0
    handoff = {"device_view": {"call": "blub_fluid_view", "bytes_copied": 0, "ms": round(t_view * 1e3, 4)},
               "host_download_positions": {"call": "blub_fluid_download(BLUB_TAP_PARTICLE_POS)", "bytes": int(pos.nbytes), "ms": round(t_dl * 1e3, 3),
                                           "note": "pageable destination; not part of the step, not in e2e"}}
    del np
    return phases, in_step, handoff, steps_done


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from oracle import oracle as O

    sc, desc = workload_desc(args.workload)
    n = max(1, args.gpus)
    if n == 1:
        f = O.fluid_from_scene(O.load_scene(scene_path(workload_scene(args.workload))))
    else:  # the same stacked scene the sharded arm simulates on n GPUs (value = n * steps/s, i.e. slab-steps/s)
        import numpy as np

        d, scale = sc["fluid"]["grid_dimension"], np.float32(sc["fluid"]["grid_to_world_scale"])
        f = O.OracleFluid(d["x"], d["y"], d["z"] * n, int(sc["fluid"]["max_num_particles"]) * n)
        f.add_fluid_cube([0.0, 0.0, 0.0], [d["x"] / 2.0, d["y"] / 4.0, float(d["z"] * n)])
        f.set_gravity_grid([np.float32(sc["gravity"][c]) / scale for c in "xyz"])
        desc = f"{n} z-slabs of {d['x']}x{d['y']}x{d['z']} cells = {d['x']}x{d['y']}x{d['z'] * n} grid, z-uniform dam (x < {d['x'] // 2}, y < {d['y'] // 4})"
    # bounded sample: one CPU step of the 256^3 workload takes seconds, so time as many of the K requested steps as fit
    # into the budget (at least one) after at most one untimed step
    budget = float(os.environ.get("BLUB_REF_BUDGET_S", "150"))
    step = oracle_stepper(f, sc, args.workload) if n == 1 else (lambda: f.step(O.DT_120HZ))
    for _ in range(min(args.warmup, 1)):
        step()
    t0 = time.perf_counter()
    timed = 0
    while timed < args.steps:
        step()
        timed += 1
        if time.perf_counter() - t0 > budget:
            break
    t = time.perf_counter() - t0
    v = n * timed / t
    cores = os.cpu_count() or 1
    line = {"impl": "reference", "metric": METRIC, "value": round(v, 5), "unit": "steps/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": round(1e3 * t / timed, 3), "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": config_block(desc, f.num_particles, O.DT_120HZ, f"CPU restatement of the reference (oracle/), OpenMP over {cores} host threads; the wgpu reference cannot run here",
                                   f"{timed} step(s) after {min(args.warmup, 1)} untimed"),
            "cpu_baseline": {"value": round(v, 5), "unit": "steps/s", "cores": cores, "kind": "port",
                             "sample": f"{timed} of the {args.steps} requested step(s) of {args.workload} timed ({budget:.0f} s budget), after {min(args.warmup, 1)} untimed"},
            "e2e": {"value": round(v, 5), "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=None)
    ap.add_argument("--impl", default="blub", choices=["blub", "reference"])
    ap.add_argument("--workload", default="dam_256")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--no-sharded-pcg", action="store_true")
    ap.add_argument("--no-scaling-reference", action="store_true")
    ap.add_argument("--no-phases", action="store_true", help="skip the late-window timing and the in-step stage / roofline analysis (N = 1)")
    ap.add_argument("--late-start", type=int, default=100, help="first step of the late timing window (N = 1)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the fluid state they produced to DIR/<name>.npy (float32, seeded samples, <= 64 MB)")
    ap.add_argument("--multi", default="sharded", choices=["sharded", "stacked", "split", "replicas"],
                    help="N > 1: one z-slab sharded simulation of a z-uniform dam (default: weak scaling, balanced), of N stacked dam_256 cubes, of the workload's "
                         "OWN grid cut into N slabs (split: strong scaling, e.g. --workload basin_512 = config C4), or N independent replicas")
    args = ap.parse_args()
    if args.impl == "reference":
        args.steps = args.steps if args.steps is not None else 2
        args.warmup = args.warmup if args.warmup is not None else 1
        return run_reference(args)
    args.steps = args.steps if args.steps is not None else 100
    args.warmup = args.warmup if args.warmup is not None else 10

    import torch
    import torch.distributed as dist

    import blub_b200
    from blub_b200 import fluid as F

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs an H100: no CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    sc, desc = workload_desc(args.workload)
    dt = F.DT_120HZ
    has_solid = args.workload in SOLID_WORKLOADS
    if has_solid and world > 1:
        args.multi = "replicas"  # the moving-solid workload is not sharded: N independent replicas
    sharded_step = world > 1 and args.multi in ("sharded", "stacked", "split")
    if not sharded_step:
        fluid = blub_b200.HybridFluid.from_scene(scene_path(workload_scene(args.workload)), device=local)
        npart = fluid.num_particles
        parallelism = "single GPU" if world == 1 else f"{world} independent replicas (one scene per GPU, no exchange)"
    else:
        # Weak scaling of ONE simulation: `world` copies of the workload stacked along z in a single connected domain, one
        # z-slab (= one copy's worth of grid and particles) per GPU; particles migrate and halos are exchanged across the faces.
        from blub_b200 import slab

        d = sc["fluid"]["grid_dimension"]
        scale = sc["fluid"]["grid_to_world_scale"]
        split = args.multi == "split"  # STRONG scaling: the workload's own grid cut into `world` z-slabs (C4 = basin_512 on 8 GPUs; dam_256 literally)
        if split and (d["z"] % world or (d["z"] // world) % 4):
            raise SystemExit(f"--multi split: {d['z']} planes cannot be cut into {world} slabs of whole 4-plane tiles")
        nz_owned = d["z"] // world if split else d["z"]
        cap = int(sc["fluid"]["max_num_particles"] * 2) // (world if split else 1)  # head room: fluid flows between slabs
        if split and args.workload == "dam_256":
            cap = int(sc["fluid"]["max_num_particles"])  # the dam starts inside the first half of the slabs
        fluid = blub_b200.HybridFluid.create_slab(d["x"], d["y"], nz_owned, cap, rank=rank, world=world, device=local)
        handles = slab.exchange_handles(fluid.ipc_export_window(), dist)
        own = fluid.slab_window()[0]
        fluid.attach_slab_peers([own if k == rank else F.ipc_open(handles[k], local) for k in range(world)])
        if args.multi == "sharded":
            # balanced weak-scaling scene: the dam is uniform along z (x < 128, y < 64 cells, every plane), so the break runs in
            # the x-y plane and no slab gains or loses fluid: per-GPU work really is fixed (16.3 M particles per slab, as in
            # dam_256).  `--multi stacked` stacks N copies of the dam_256 cube instead; they drain towards z = 0 and unbalance.
            zmax = float(d["z"] * world)
            fluid.add_fluid_cube([0.0, 0.0, 0.0], [d["x"] / 2.0, d["y"] / 4.0, zmax])
        elif split:
            for cube in sc["fluid"]["fluid_cubes"]:  # global coordinates: every rank keeps the particles of its planes
                fluid.add_fluid_cube([cube["min"][c] / scale for c in "xyz"], [cube["max"][c] / scale for c in "xyz"])
        else:
            for k in range(world):
                for cube in sc["fluid"]["fluid_cubes"]:
                    mn = [cube["min"][c] / scale for c in "xyz"]
                    mx = [cube["max"][c] / scale for c in "xyz"]
                    mn[2] += k * d["z"]
                    mx[2] = min(mx[2], d["z"] - 1) + k * d["z"]
                    fluid.add_fluid_cube(mn, mx)
        fluid.set_gravity_grid([sc["gravity"][c] / scale for c in "xyz"])
        counts = [None] * world
        dist.all_gather_object(counts, fluid.num_particles)
        npart = sum(counts)
        if split:
            desc = f"{desc}, cut into {world} z-slabs of {nz_owned} planes (strong scaling)"
        elif args.multi == "sharded":
            desc = f"{world} z-slabs of {d['x']}x{d['y']}x{d['z']} cells = {d['x']}x{d['y']}x{d['z'] * world} grid, z-uniform dam (x < {d['x'] // 2}, y < {d['y'] // 4})"
        else:
            desc = f"{world} x ({desc}) stacked along z = {d['x']}x{d['y']}x{d['z'] * world} grid"
        parallelism = f"one simulation on {world} z-slabs (P2P halo exchange + particle migration, in-kernel PCG exchange)"
    stepper = SolidStepper(fluid, sc, SOLID_WORKLOADS[args.workload]["solid"], local) if has_solid else None
    step = stepper.step if stepper else fluid.step
    for _ in range(max(args.warmup, 3)):
        step(dt)
    fluid.synchronize()

    # ---- device-timed region: K steps between CUDA events on the fluid's stream, barrier + sync on both sides --------
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = blub_b200.kernel_launch_count()
    ms = stepper.time_steps(dt, args.steps) if stepper else fluid.time_steps(dt, args.steps)
    launches = blub_b200.kernel_launch_count() - launches0
    barrier()
    clocks = sampler.stop() if rank == 0 else None
    dumped = None
    if args.dump_outputs:  # the state after the last timed step, before anything else advances the simulation
        dumped = dump_outputs(fluid, args.dump_outputs, f"_rank{rank}" if world > 1 else "", parts=world)
    t_ms = torch.tensor([ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t_ms, op=dist.ReduceOp.MAX)
    ms_max = float(t_ms.item())

    # ---- end-to-end through the C ABI: per step one pinned H2D parameter block, one 16-byte D2H statistics read, host sync --
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step(dt)
        fluid.synchronize()
        fluid.update_statistics()
    fluid.synchronize()
    e2e_s = time.perf_counter() - t0
    t_e = torch.tensor([e2e_s], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t_e, op=dist.ReduceOp.MAX)
    e2e_s = float(t_e.item())
    stats = fluid.pressure_solver_stats(0)[-1], fluid.pressure_solver_stats(1)[-1]
    steps_done = max(args.warmup, 3) + 2 * args.steps
    scene_phases = in_step = handoff = None
    if world == 1 and not args.no_phases:
        scene_phases, in_step, handoff, steps_done = late_window_and_in_step(fluid, step, stepper, dt, steps_done, args, ms / args.steps)
    slab_err = fluid.slab_error() if sharded_step else 0
    slab_counts = None
    if sharded_step:
        info = [None] * world
        dist.all_gather_object(info, (fluid.num_particles, slab_err))
        slab_counts = [c for c, _ in info]
        slab_err = max(e for _, e in info)
    if world > 1:
        dist.barrier()
    fluid.close()

    sharded = None
    if world > 1 and not args.no_sharded_pcg:
        sharded = pcg_sharded(rank, world, local)
    scaling_ref = None
    if world == 1 and not args.no_scaling_reference:
        d = sc["fluid"]["grid_dimension"]
        g1 = blub_b200.HybridFluid(d["x"], d["y"], d["z"], sc["fluid"]["max_num_particles"], device=local)
        g1.add_fluid_cube([0.0, 0.0, 0.0], [d["x"] / 2.0, d["y"] / 4.0, float(d["z"])])
        g1.set_gravity_grid([sc["gravity"][c] / sc["fluid"]["grid_to_world_scale"] for c in "xyz"])
        for _ in range(max(args.warmup, 3)):
            g1.step(dt)
        g1.synchronize()
        ms1 = g1.time_steps(dt, args.steps)
        scaling_ref = {"workload": f"z-uniform dam (x < {d['x'] // 2}, y < {d['y'] // 4}) on one {d['x']}x{d['y']}x{d['z']} grid: the per-slab scene of the N > 1 runs",
                       "particles": g1.num_particles, "value": round(args.steps / (ms1 * 1e-3), 3), "unit": "steps/s"}
        g1.close()
    roof = cpu = None
    if rank == 0 and not args.no_roofline:
        roof = pcg_roofline(local)
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu = cpu_baseline_sample(args.workload, 1)
    if rank == 0:
        split_mode = sharded_step and args.multi == "split"
        steps_per_s = (1 if split_mode else world) * args.steps / (ms_max * 1e-3)
        line = {
            "metric": METRIC, "value": round(steps_per_s, 3), "unit": "steps/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": round(ms_max / args.steps, 4), "higher_is_better": True, "scaling": "strong" if split_mode else "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": config_block(desc, npart, dt, parallelism, f"steps {max(args.warmup, 3)}..{max(args.warmup, 3) + args.steps - 1} of the scene (see scene_phases for a later window)"),
            "last_solver_stats": {"velocity": stats[0], "density": stats[1]},
            "clocks": clocks,
            "e2e": {"value": round((1 if split_mode else world) * args.steps / e2e_s, 3), "unit": "steps/s", "h2d_bytes_per_step": 36, "d2h_bytes_per_step": 16,
                    "note": "blub_fluid_step + blub_fluid_synchronize + blub_fluid_update_statistics per step (host-timed); the state stays on the device as in the "
                            "reference (hybrid_fluid.rs:770): per step the host sends the 36-byte parameter block and reads the two 8-byte solver statistics; see result_handoff"},
            "gpu_launches": int(launches),
            "simulation_steps_per_s": round(args.steps / (ms_max * 1e-3), 3),
            "value_definition": ("steps/s of the one simulation" if world == 1 or split_mode or not sharded_step else
                                 f"slab-steps/s = {world} x simulation_steps_per_s: ONE simulation on {world} z-slabs, each slab a 256^3-cell, 16.3 M-particle share "
                                 "(weak scaling: the whole-job aggregate in units of the N = 1 workload)") if sharded_step or world == 1 else
                                f"{world} independent replicas x steps/s",
            "slab_error": slab_err,
            "slab_particles": slab_counts,
            "roofline": roof,
            "cpu_baseline": cpu,
        }
        if scene_phases is not None:
            line["scene_phases"] = scene_phases
        if in_step is not None:
            line["in_step"] = in_step
        if handoff is not None:
            line["result_handoff"] = handoff
        if scaling_ref is not None:
            line["scaling_reference"] = scaling_ref
        if dumped is not None:
            line["dumped_outputs"] = dumped
        if sharded is not None:
            line["pcg_sharded"] = sharded
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
