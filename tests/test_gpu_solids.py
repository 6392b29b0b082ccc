"""Analytic rigid solids (SURVEY section 8 f1 / BASELINE config 5's mechanism): the CUDA voxelizer + animation maths against
the NumPy restatement of src/scene/models.rs:154-224 and conservative_hull.frag:17-23, and a moving solid inside a step."""
import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from oracle import solids as S
from tests import util
from tests.test_gpu_parity import ROTATING_BOX, ROTATING_BOX_T
from tests.util import DT

pytestmark = pytest.mark.gpu

# parameters of scenes/#double_dam_wgpulogo_rotating.json:61-79 (translation SmoothStep over 2 s, rotation about y), applied to a box
OBJ = {"world_position": [0.44, 0.12, 0.16], "scale": 1.0, "rotation_angles": [0.0, 30.0, 10.0], "shape": "box", "half_extent": [0.06, 0.10, 0.06],
       "translation": {"target": [0.2, 0.12, 0.16], "curve": "SmoothStep", "duration": 2.0}, "rotation": {"axis": [0.0, 1.0, 0.0], "deg_per_sec": 20.0}}


@pytest.mark.parametrize("t", [0.0, 0.5, 1.7, 2.6, 4.1])
@pytest.mark.parametrize("shape", ["box", "sphere"])
def test_voxelizer_matches_numpy_restatement(t, shape):
    import torch
    dims, scale, origin = (64, 32, 32), 0.01, (0.0, 0.0, 0.0)  # the object travels between x = 44 and x = 20 cells
    obj = dict(OBJ, shape=shape)
    vol = torch.full((32, 32, 64, 4), 7.0, dtype=torch.float16, device="cuda")
    st = F.solid_voxelize(vol.data_ptr(), dims, obj, scale, origin, t, DT)
    torch.cuda.synchronize()
    got = vol.float().cpu().numpy()
    want, ref = S.voxelize(obj, dims, scale, origin, t, DT)
    assert np.allclose(np.array(st.centre_voxel), ref["centre"], atol=2e-3)
    assert np.allclose(np.array(st.velocity_voxel), ref["velocity"], atol=2e-2 * max(1.0, np.abs(ref["velocity"]).max()))
    assert np.allclose(np.array(st.axis_scaled), ref["axis"], atol=1e-6)
    assert np.allclose(np.array(st.rotation).reshape(3, 3), ref["R"], atol=1e-5)
    inside_g, inside_w = got[..., 3] > 0, want[..., 3] > 0
    # voxels whose centre sits on the surface may flip with fp32 vs fp64 rounding: allow a handful
    assert (inside_g != inside_w).sum() <= 0.01 * max(1, inside_w.sum())
    both = inside_g & inside_w
    assert both.sum() > 50
    vmax = max(1.0, np.abs(want[both, :3]).max())
    assert np.abs(got[both, :3] - want[both, :3]).max() <= 4e-3 * vmax + 2e-2  # fp16 storage
    assert (got[~inside_g] == 0).all()


def test_moving_box_in_a_step_matches_oracle():
    import torch
    orc = util.oracle_from_scene("dam_small")
    gpu = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    for f in (orc, gpu):
        f.set_rebin_frequency(0)
    util.tight_solver(orc, gpu)  # trajectory comparison: converged solves (SURVEY 8c)
    dims, scale, origin = (32, 32, 32), 0.01, (0.0, 0.0, 0.0)
    # inside the dam (fluid in x < 16): translating toward x = 5 cells and rotating about an axis that is no grid axis
    obj = ROTATING_BOX
    vol = torch.zeros((32, 32, 32, 4), dtype=torch.float16, device="cuda")
    gpu.set_solid_voxels(vol.data_ptr())
    t = ROTATING_BOX_T
    inside = []
    for _ in range(4):
        t += DT
        F.solid_voxelize(vol.data_ptr(), dims, obj, scale, origin, t, DT)  # Scene::step: voxelize, then the fluid step
        torch.cuda.synchronize()
        want, _ = S.voxelize(obj, dims, scale, origin, t, DT)
        # feed the oracle the SAME fp16-rounded volume the GPU path sees
        got = vol.float().cpu().numpy()
        orc.set_voxels(got)
        assert ((got[..., 3] > 0) != (want[..., 3] > 0)).sum() <= 8
        c = np.floor(orc.particles()[:, :3]).astype(int)
        inside.append((got[..., 3] > 0)[c[:, 2], c[:, 1], c[:, 0]].sum())
        orc.step(DT)
        gpu.step(DT)
        faces, near = util.solid_contact(orc.grid(O.ARR_MARKER), got, orc.particles())  # the marker and particles of the step this volume moved
        assert faces >= 250 and near >= 5000, (faces, near)
        gpu.synchronize()
        util.markers_agree(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER))
        p_o = orc.particles()[:, :3].copy()
        d = np.abs(p_o - gpu.download_particles()[:, :3]).max(axis=1)
        assert np.quantile(d, 0.999) <= 1e-2, (np.quantile(d, 0.999), d.max())
        # one step at a time: particles the box pushes around inside it take branches that amplify round-off over several steps, so every step
        # starts the CUDA fluid from the oracle's particles
        gpu.set_particles(np.c_[p_o, np.zeros(len(p_o), np.float32)], orc.particles(O.ARR_ROWX), orc.particles(O.ARR_ROWY), orc.particles(O.ARR_ROWZ))
    solid = (vol[..., 3] > 0).cpu().numpy()
    now = []
    for p in (gpu.download_particles()[:, :3], orc.particles()[:, :3]):
        c = np.floor(p).astype(int)
        now.append(solid[c[:, 2], c[:, 1], c[:, 0]].sum())
    # the box starts with thousands of particles inside; the moving wall pushes them out one cell per step (advect_particles.comp:45-64),
    # equally in both implementations
    assert inside[0] > 4000 and now[0] < 0.5 * inside[0] and abs(int(now[0]) - int(now[1])) <= 0.001 * orc.num_particles, (inside, now)
