"""Full-size (BASELINE.json configs) property checks on the H100: things the oracle is too slow for."""
import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import util
from tests.util import DT

pytestmark = pytest.mark.gpu


def divergence(gpu):
    m = gpu.download_grid(F.TAP_MARKER)
    ux, uy, uz = gpu.download_grid(F.TAP_UX), gpu.download_grid(F.TAP_UY), gpu.download_grid(F.TAP_UZ)
    div = np.zeros_like(ux)
    div[1:, 1:, 1:] = (ux[1:, 1:, 1:] - ux[1:, 1:, :-1]) + (uy[1:, 1:, 1:] - uy[1:, :-1, 1:]) + (uz[1:, 1:, 1:] - uz[:-1, 1:, 1:])
    return div, m


@pytest.mark.parametrize("name,count", [("dam_halfhalf", 1218672), ("dam_halfhalf_highres", 10113264)])
def test_scene_runs_conserves_particles_and_projects(name, count):
    gpu = blub_b200.HybridFluid.from_scene(util.scene_path(name))
    assert gpu.num_particles == count
    for _ in range(2):
        gpu.step(DT)
    # tight projection on the 3rd step: divergence on fluid cells must drop below the solver tolerance
    gpu.set_solver_config(0, 1e-2, 4000, 8)
    gpu.step_stages(DT, 0, 5)
    err, it = gpu.last_solve(0)
    assert 0 < it < 4000, (err, it)
    div, m = divergence(gpu)
    fluid = m == 1
    interior = fluid.copy()
    for ax in range(3):  # cells with only fluid/air neighbours: plain divergence is the solver's residual there
        interior &= np.roll(m, 1, ax) != 0
        interior &= np.roll(m, -1, ax) != 0
    assert err < 1e-2 / DT and np.abs(div[interior]).max() <= 1.05 * err + 1e-3, (err, it, np.abs(div[interior]).max())
    gpu.step_stages(DT, 5, 14)
    p = gpu.download_particles()[:, :3]
    assert p.shape[0] == count and np.isfinite(p).all()
    lo, hi = 1.001 - 1e-5, np.array([gpu.nx, gpu.ny, gpu.nz]) - 1.001 + 1e-4
    assert (p >= lo).all() and (p <= hi).all()


def test_256_cubed_step_and_binning():
    gpu = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    assert gpu.num_particles == 16387064
    before = gpu.download_particles()[:, :3]
    gpu.set_rebin_frequency(1)
    gpu.step(DT)
    gpu.synchronize()
    after = gpu.download_particles()[:, :3]
    assert after.shape == before.shape and np.isfinite(after).all()
    # rest density ~ 8 per cell in the bulk
    c = np.floor(after).astype(np.int64)
    key = (c[:, 2] * gpu.ny + c[:, 1]) * gpu.nx + c[:, 0]
    counts = np.bincount(key, minlength=gpu.n).reshape(gpu.nz, gpu.ny, gpu.nx)
    bulk = counts[8:120, 8:100, 8:120]
    assert 7.5 < bulk.mean() < 8.5
    e, it = gpu.last_solve(0)
    assert it % 4 == 0 and 4 <= it <= 32
