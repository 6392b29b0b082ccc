"""Flow kernel time of tap_256 on steps that drain nothing and on steps that drain (torch.profiler), and the per-stage time of one eager
step of dam_256 and tap_256 at step 31.  Results: profiles/h100_flow.json.  Run from the repository root after python -m blub_b200.build."""
import torch, numpy as np, blub_b200
from torch.profiler import profile, ProfilerActivity
from tests import util
DT = util.DT
NAMES = ("flow_count_kernel", "flow_compact_kernel", "flow_copy_back_kernel", "flow_need_kernel", "flow_emit_kernel", "scan_")
def prof(f, steps=5):
    f.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as p:
        for _ in range(steps): f.step(DT)
        f.synchronize()
    tot = {}
    for e in p.events():
        for n in NAMES:
            if n in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                tot[n] = tot.get(n, 0) + e.device_time_total
    return {k: round(v / steps / 1000, 4) for k, v in tot.items()}
src = [((179, 199, 99), (199, 209, 139), (0, -200, 0))]
f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_256"))
for _ in range(3): f.step(DT)
c0 = f.flow_counters
print("no drain reached (steps 4-8):", prof(f), "ms/step", f.flow_counters, f.num_particles)
f.set_flow(sources=src, drains=[((100, 1, 1), (128, 6, 128))])  # inside the dam block's floor: drains every step
c1 = f.flow_counters
print("drain inside the block (steps 9-13):", prof(f), "ms/step", "drained per step", (f.flow_counters["drained"] - c1["drained"]) / 5, f.num_particles)
# per-stage time of one eager step at the same step index, dam_256 against tap_256
for name in ("dam_256", "tap_256"):
    g = blub_b200.HybridFluid.from_scene(util.scene_path(name))
    for _ in range(30): g.step(DT)
    ms = [g.step_timed(DT) for _ in range(3)]
    print(name, "step 31-33 stage ms", [round(float(np.median([m[s] for m in ms])), 3) for s in range(14)], "total", round(float(np.median([sum(m) for m in ms])), 3),
          "particles", g.num_particles, "last solve iterations", g.last_solve(0)[1], g.last_solve(1)[1])
    del g
