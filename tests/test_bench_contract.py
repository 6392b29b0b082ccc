"""bench.py contract checks that need no GPU: the reference arm (CPU restatement) prints one JSON line with the keys the
driver reads, for N = 1 and for the sharded scene of an N > 1 run."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("gpus", [1, 2])
def test_reference_arm_prints_one_json_line(gpus):
    env = dict(os.environ, BLUB_REF_BUDGET_S="20")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "dam_small", "--gpus", str(gpus),
                          "--steps", "2", "--warmup", "1"], capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["metric"] == "simulation steps/sec" and j["unit"] == "steps/s"
    assert j["n_gpus"] == gpus and j["higher_is_better"] is True and j["value"] > 0
    assert j["cpu_baseline"]["kind"] == "port" and j["cpu_baseline"]["value"] == j["value"] and j["cpu_baseline"]["cores"] >= 1
    assert j["e2e"] == {"value": j["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in j["config"]


def test_gpu_arm_refuses_to_run_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=300)
    assert out.returncode != 0 and "no CUDA device" in (out.stderr + out.stdout)


class _StubFluid:
    """Stands in for HybridFluid: deterministic arrays of the shapes the taps return."""

    def __init__(self, nparticles, dims):
        self.num_particles, (self.nx, self.ny, self.nz) = nparticles, dims
        self.n = self.nx * self.ny * self.nz

    def synchronize(self):
        pass

    def download_particles(self, tap=0):
        import numpy as np
        return (np.arange(self.num_particles * 4, dtype=np.float32).reshape(-1, 4) + tap)

    def download_grid(self, tap):
        import numpy as np
        a = np.arange(self.n, dtype=np.float32).reshape(self.nz, self.ny, self.nx) + tap
        return a.astype(np.int8) if tap == 7 else a


def test_dump_outputs_writes_float_arrays_within_64_mb(tmp_path):
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    info = bench.dump_outputs(_StubFluid(16_387_064 // 8, (256, 256, 256)), str(tmp_path / "a"))
    again = bench.dump_outputs(_StubFluid(16_387_064 // 8, (256, 256, 256)), str(tmp_path / "b"))
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == sorted(os.listdir(tmp_path / "b")) and len(files) == 12
    total = 0
    for f in files:
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), f  # same inputs, same seeded sample
        total += os.path.getsize(tmp_path / "a" / f)
    assert total <= 64 * 2 ** 20 and info.pop("dir") != again.pop("dir") and info == again and info["cells_dumped"] == bench.DUMP_CELLS
    pi = np.load(tmp_path / "a" / "particle_index.npy").astype(np.int64)
    assert np.array_equal(np.load(tmp_path / "a" / "particles_position.npy")[:, 0], pi * 4)


def test_dump_outputs_of_eight_ranks_stay_within_64_mb(tmp_path):
    sys.path.insert(0, ROOT)
    import bench
    for rank in range(8):  # eight z-slab ranks of the sharded 256^3 bench, one directory
        bench.dump_outputs(_StubFluid(16_387_064 // 8, (256, 256, 256 + 8)), str(tmp_path), f"_rank{rank}", parts=8)
    files = os.listdir(tmp_path)
    assert len(files) == 8 * 12 and sum(os.path.getsize(tmp_path / f) for f in files) <= 64 * 2 ** 20


def test_dump_outputs_keeps_small_arrays_whole(tmp_path):
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    bench.dump_outputs(_StubFluid(1000, (32, 32, 32)), str(tmp_path))
    assert np.load(tmp_path / "particles_velocity_x.npy").shape == (1000, 4)
    assert np.array_equal(np.load(tmp_path / "cell_index.npy"), np.arange(32 ** 3))


@pytest.mark.gpu
def test_bench_dump_outputs_on_the_gpu(tmp_path):
    """Two runs with the same arguments dump the same outputs, bit for bit; --steps sets how many steps are timed (the kernel launches
    of the timed region scale with it, and the dumped state is a different one after 10 steps)."""
    import numpy as np
    dirs, lines = [tmp_path / "a", tmp_path / "b", tmp_path / "c"], []
    for d, steps in zip(dirs, (20, 20, 10)):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "dam_small", "--steps", str(steps), "--warmup", "3",
                              "--no-cpu-baseline", "--no-roofline", "--no-scaling-reference", "--no-phases", "--dump-outputs", str(d)],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]
        j = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
        assert j["dumped_outputs"]["particles"] == j["config"]["particles"]
        lines.append(j)
    launches = [l["gpu_launches"] for l in lines]
    assert launches[0] == launches[1] >= 20 * 20 and 1.8 <= launches[0] / launches[2] <= 2.2, launches
    assert not np.array_equal(np.load(dirs[0] / "particles_position.npy"), np.load(dirs[2] / "particles_position.npy"))
    dirs = dirs[:2]
    pos = np.load(dirs[0] / "particles_position.npy")
    assert pos.dtype == np.float32 and pos.shape == (j["config"]["particles"], 4) and np.isfinite(pos).all()
    assert np.load(dirs[0] / "pressure_from_density.npy").shape == (32 ** 3,)
    names = sorted(os.listdir(dirs[0]))
    assert names == sorted(os.listdir(dirs[1])) and len(names) == 12
    for name in names:
        assert np.array_equal(np.load(dirs[0] / name), np.load(dirs[1] / name)), name
