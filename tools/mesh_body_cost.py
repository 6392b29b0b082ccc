"""What triangle-mesh bodies cost on dam_256 (256^3 grid, 16.4 M particles): steps/s of a fluid without bodies, of one with four analytic bodies
(two boxes, two spheres) and of one with four mesh bodies (three icospheres at subdivision 4, 5120 triangles each, and a torus of 8192
triangles), 3 x 100 steps each, alternating in one process (the order alternates too).  Then, in runs of their own under torch.profiler, the
device time per step of every body kernel and of the bit-volume memset for the four mesh bodies, and for a 12-triangle box mesh of side 40
cells, whose faces each cover about 1600 cell rows: the case where one triangle has the most rows to walk.  Reads the card name and power
limit in the same run.  Last, the hollow hull of tests/test_gpu_mesh_bodies.py (outer side 20 cells, walls and floor 2 thick, solid volume
3392 cells) at relative densities whose mass / outer volume is 0.64, 0.85 and 0.95 in a 64^3 tank filled to 32 cells: the mean draft
and bottom height over the last 100 of 400 steps, which shows where it stops floating.  Run from the repository root after python -m blub_b200.build:

    python tools/mesh_body_cost.py [--out profiles/h100_mesh_bodies.json]
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
from tests import body_ref, mesh_body_ref as M, util  # noqa: E402

DT = util.DT
ANALYTIC = [body_ref.body("box", (12, 8, 10), 0.5, (64, 120, 64)), body_ref.body("box", (6, 6, 16), 2.0, (190, 60, 190), (0.9659258, 0.0, 0.2588190, 0.0)),
            body_ref.body("sphere", 10, 0.8, (128, 90, 200)), body_ref.body("sphere", 14, 1.2, (200, 150, 60))]
ICO4, TORUS = M.icosphere(4, 1.0), M.torus(2.0, 0.8, 128, 32)
MESHES = [(ICO4, 10.0, body_ref.body("box", 1, 0.5, (64, 120, 64))), (ICO4, 12.0, body_ref.body("box", 1, 2.0, (190, 60, 190))),
          (ICO4, 10.0, body_ref.body("box", 1, 0.8, (128, 90, 200))), (TORUS, 6.0, body_ref.body("box", 1, 1.2, (200, 150, 60), (0.9659258, 0.0, 0.2588190, 0.0)))]
BIG_BOX = [(M.box_mesh((-20, -20, -20), (20, 20, 20)), 1.0, body_ref.body("box", 1, 0.5, (128, 100, 128), (0.9659258, 0.0, 0.2588190, 0.0)))]
NAMES = ("mesh_body_transform_kernel", "mesh_body_cross_kernel", "mesh_body_parity_kernel", "body_composite_kernel", "body_load_kernel",
         "body_integrate_kernel", "Memset")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def mesh_dicts(spec):
    return [dict(b, shape="mesh", mesh=mesh, scale=s) for mesh, s, b in spec]


def device_ms_per_step(f, steps=10):
    """torch.profiler device time per step of the body kernels and memsets over `steps` eagerly launched steps."""
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


def hull_run(rho, steps=400, keep=100):
    from tests.test_gpu_bodies import surface
    from tests.test_gpu_loads import seed_around
    from blub_b200 import fluid as F
    pos, tri = M.hollow_box(20, 2)
    f = blub_b200.HybridFluid(64, 64, 64, 8 * 64 * 64 * 32)
    f.set_gravity_grid((0.0, -981.0, 0.0))
    lo = (22, 20, 22)
    seed_around(f, 33, lo, (42, 33, 42))
    for which in (0, 1):
        f.set_solver_config(which, 1e-5, 4000, 4)
    f.set_bodies(mesh_dicts([((pos, tri), 1.0, body_ref.body("box", 1, rho, lo))]))
    vmin = float(F.mesh_body_vertices(pos, tri, 1.0)[:, 1].min())
    drafts, bottoms = [], []
    for step in range(steps):
        f.step(DT)
        if step >= steps - keep:
            b = f.bodies()[0]
            bottom = b["centre"][1] + vmin
            bottoms.append(bottom)
            drafts.append(surface(f.download_grid(F.TAP_MARKER), b["centre"][0], b["centre"][2]) - bottom)
    V = f.body_mass_properties(0)["volume"]
    return {"relative_density": rho, "mass_over_outer_volume": round(rho * V / 8000, 3), "mean_draft": round(sum(drafts) / len(drafts), 3),
            "predicted_draft": round(rho * V / 400 - 1.0, 3), "bottom_min": round(min(bottoms), 3), "bottom_max": round(max(bottoms), 3)}


def progress(*what):
    print(*what, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("profiles", "h100_mesh_bodies.json"))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    scene = util.scene_path("dam_256")
    fluids = {name: blub_b200.HybridFluid.from_scene(scene) for name in ("no_bodies", "four_analytic_bodies", "four_mesh_bodies")}
    fluids["four_analytic_bodies"].set_bodies(ANALYTIC)
    fluids["four_mesh_bodies"].set_bodies(mesh_dicts(MESHES))
    for f in fluids.values():
        f.step(DT)  # step 0 (rebinning) and the graph captures
        f.time_steps(DT, 9)
    rates = {k: [] for k in fluids}
    for r in range(args.rounds):
        for name, f in (list(fluids.items()) if r % 2 == 0 else list(fluids.items())[::-1]):
            rates[name].append(round(args.steps / (f.time_steps(DT, args.steps) / 1000.0), 2))
            progress(name, rates[name][-1], "steps/s")
    f = fluids["four_mesh_bodies"]
    h = [f.body_history(i) for i in range(len(MESHES))]
    last_pose = [{"step": int(v["step"][-1]), "centre": v["centre"][-1].tolist(), "velocity": v["velocity"][-1].tolist(),
                  "wetted_faces": int(v["wetted_faces"][-1])} for v in h]
    kernels = {"four_mesh_bodies": device_ms_per_step(f)}
    progress("four_mesh_bodies", kernels["four_mesh_bodies"])
    f = None
    fluids.clear()  # frees the three dam_256 fluids before the next one
    big = blub_b200.HybridFluid.from_scene(scene)
    big.set_bodies(mesh_dicts(BIG_BOX))
    big.step(DT)
    kernels["box_mesh_40_cells"] = device_ms_per_step(big)
    progress("box_mesh_40_cells", kernels["box_mesh_40_cells"])
    particles = big.num_particles
    del big
    hull = []
    for rho in (1.5, 2.0, 2.25):
        hull.append(hull_run(rho))
        progress("hollow hull", hull[-1])
    out = {
        "card": card(),
        "workload": "dam_256",
        "particles": particles,
        "mesh_bodies": [{"triangles": int(len(m[0][1])), "vertices": int(len(m[0][0])), "scale": m[1], "placement": m[2]} for m in MESHES],
        "analytic_bodies": ANALYTIC,
        "steps_per_round": args.steps,
        "steps_per_s": rates,
        "device_ms_per_step": kernels,
        "last_pose": last_pose,
        "hollow_hull": hull,
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
