"""GPU: the brick schedule of the density and P2G scatters (transfer_kernels.cu, DESIGN.md §3.2) changes no bit.  Every case runs twice in fresh
processes, once as built and once with BLUB_SCATTER_SCHEDULE=off (read once per process: the scatter then walks the 256-particle chunks
only), and the density rhs, the P2G velocities and marker and the particles must be equal bit for bit.  20 steps span the
re-sorts of steps 0, 8 and 16; a fluid loaded from a state file runs the chunks until its next re-sort.  The P2G scatter walks the work items
only when they fill several waves of resident blocks, which the small scenes do not: the dam_256 case (16.4 M particles) covers that path over
steps 0-9, 56, 57 and 230, and crowded_items (BLUB_P2G_ITEM_WAVES=0) on bricks that hold several work items each.
Arrays are compared by their SHA-256 digests."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 20


def _fluid(name):
    import blub_b200
    from tests import util

    return blub_b200.HybridFluid.from_scene(util.scene_path(name))


def _crowded():
    """60,000 particles piled into 4 x 4 x 4 cells of a 48^3 grid: one brick holds far more than one work item of warps."""
    import blub_b200

    rng = np.random.default_rng(5)
    pos = np.zeros((60000, 4), np.float32)
    pos[:, :3] = rng.uniform(20.0, 24.0, (60000, 3))
    f = blub_b200.HybridFluid(48, 48, 48, 80000)
    f.set_particles(pos, *[rng.standard_normal((60000, 4)).astype(np.float32) * 0.1 for _ in range(3)])
    return f


def run_case(case, tmp):
    """The arrays a case records, step by step."""
    import blub_b200.fluid as F
    from tests.util import DT

    out = {}

    def record(f, k, what):
        f.synchronize()
        for name, tap in what:
            a = f.download_grid(tap) if tap != F.TAP_POS else f.download_particles(tap)
            out[f"{k}_{name}"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)

    p2g = (("ux", F.TAP_UX), ("uy", F.TAP_UY), ("uz", F.TAP_UZ), ("marker", F.TAP_MARKER))
    end = (("pos", F.TAP_POS), ("ux_end", F.TAP_UX))
    if case in ("eager", "crowded", "crowded_items", "dam_256"):
        # stage by stage: the P2G result after stage 0, the density rhs (the solver residual) after stage 9
        f = {"eager": lambda: _fluid("dam_small"), "crowded": _crowded, "crowded_items": _crowded, "dam_256": lambda: _fluid("dam_256")}[case]()
        f.set_graph_replay(False)
        # dam_256: the re-sorts of steps 0 and 8, then step 56 (the most decayed order of the window of step 48), 57 (the first P2G on the
        # schedule of step 56) and 230 (the step bench.py times stage by stage); the steps in between are not recorded
        checked = range(STEPS) if case != "dam_256" else [*range(10), 56, 57, 230]
        for k in range(checked[-1] + 1):
            if k not in checked:
                f.step(DT)
                continue
            f.step_stages(DT, 0, 1)
            record(f, k, p2g)
            f.step_stages(DT, 1, 10)
            record(f, k, (("rhs", F.TAP_RESIDUAL),))
            f.step_stages(DT, 10, 14)
        record(f, "end", (("pos", F.TAP_POS),))
    elif case in ("graph", "tap", "norebin"):
        f = _fluid("tap_small" if case == "tap" else "dam_small")
        if case == "norebin":
            f.set_rebin_frequency(0)
        for k in range(STEPS):
            f.step(DT)
            record(f, k, end)
        out["flow"] = np.array([f.flow_counters[k] for k in ("emitted", "drained", "refused")] if case == "tap" else [])
    elif case == "resume":
        import blub_b200

        f = _fluid("dam_small")
        for k in range(11):  # saved in the middle of the sort window of step 8
            f.step(DT)
        path = os.path.join(tmp, "mid.blub")
        f.save_state(path)
        f.close()
        g = blub_b200.HybridFluid.from_state(path)
        for k in range(11, STEPS):
            g.step(DT)
            record(g, k, end)
    else:
        raise ValueError(case)
    return out


def _run(case, tmp_path, schedule):
    out = str(tmp_path / f"{case}_{schedule}.npz")
    env = dict(os.environ)
    env.pop("BLUB_P2G_ITEM_WAVES", None)
    if case == "crowded_items":  # P2G walks the work items whenever the schedule is valid, as at millions of particles
        env["BLUB_P2G_ITEM_WAVES"] = "0"
    if schedule == "off":
        env["BLUB_SCATTER_SCHEDULE"] = "off"
    else:
        env.pop("BLUB_SCATTER_SCHEDULE", None)
    res = subprocess.run([sys.executable, "-m", "tests.test_gpu_scatter_schedule", case, out, str(tmp_path)], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    return dict(np.load(out))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["eager", "graph", "tap", "resume", "norebin", "crowded", "crowded_items", "dam_256"])
def test_schedule_changes_no_bit(case, tmp_path):
    a, b = _run(case, tmp_path, "on"), _run(case, tmp_path, "off")
    assert sorted(a) == sorted(b) and len(a) > 0
    for name in a:
        assert a[name].shape == b[name].shape and np.array_equal(a[name], b[name]), name
    if case == "tap":
        assert a["flow"][0] > 0 and a["flow"][1] > 0  # the sources emitted and the drains removed particles


if __name__ == "__main__":
    case, dst, tmp = sys.argv[1:4]
    np.savez(dst, **run_case(case, tmp))
