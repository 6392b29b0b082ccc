"""The block-private accumulator tiles of the P2G and density scatters (transfer_kernels.cu): a tile keeps every 64-bit fixed-point sum as two
32-bit words (native shared-memory atomics on sm_90a) and flushes it into the global volumes with one 64-bit reduction.  Integer sums do not
depend on how the contributions are split between tile and global path, so the scatters must give the same bits as an untiled scatter that
adds every (peer group, face) integer straight into the global volumes.  The hashes below were recorded with that untiled scatter."""
import hashlib

import numpy as np
import pytest

M32 = 0xFFFFFFFF


def tile_sum(values, order):
    """tile_add of transfer_kernels.cu, emulated word by word: low word by a 32-bit atomic add that returns the old value, the carry of
    that add plus the high half of the value into the high word."""
    lo = hi = 0
    for q in (int(values[k]) for k in order):
        ql = q & M32
        old = lo
        lo = (old + ql) & M32
        h = (((q >> 32) & M32) + (1 if lo < old else 0)) & M32
        if h:
            hi = (hi + h) & M32
    s = (hi << 32) | lo
    return s - (1 << 64) if s >> 63 else s


def test_split_word_accumulator_equals_the_int64_sum_in_any_order():
    rng = np.random.default_rng(11)
    for trial in range(300):
        n = int(rng.integers(1, 200))
        scale = [2 ** 31, 2 ** 40, 2 ** 62][trial % 3]  # within one word, weights (40 fractional bits), near the int64 range
        v = rng.integers(-scale, scale, n, dtype=np.int64)
        if trial % 5 == 0:
            v = np.abs(v) | np.int64(0xFFFFFF00)  # low words close to 2^32: almost every add wraps
        want = int(v.astype(np.uint64).sum(dtype=np.uint64).view(np.int64))  # two's complement sum modulo 2^64
        for _ in range(3):
            assert tile_sum(v, rng.permutation(n)) == want


def test_tiles_cut_the_global_reductions_of_a_sorted_dam_break():
    """The design argument for the tiles, on the oracle's dam break (32^3, 40 k particles) in the array order the CUDA path keeps (stable sort
    by primal cell every 8 steps), with the kernels' chunk (256) and tile sizes (1184 faces, 2048 cells): at every step the tiled scatters
    issue at most 35 % of the global reductions the peer groups alone issue, flushes included."""
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
    import red_stats as R

    from oracle import oracle as O
    from tests import util

    f = util.oracle_from_scene("dam_small")
    f.set_rebin_frequency(0)
    dims = O.load_scene(util.scene_path("dam_small"))["fluid"]["grid_dimension"]
    nx, ny = dims["x"], dims["y"]
    order = np.arange(f.num_particles)
    for step in range(10):
        p = f.particles()[:, :3].copy()
        if step % 8 == 0:
            order = R.sort_by_primal_cell(p, order, nx, ny)
        v, d = R.reductions_per_particle(p[order], nx, ny), R.reductions_per_particle(p[order], nx, ny, comps=(3,))
        tv, _, _ = R.tiled_global_reductions(p[order], nx, ny, 256, 1184)
        td, _, _ = R.tiled_global_reductions(p[order], nx, ny, 256, 2048, comps=(3,))
        assert tv <= 0.35 * 2 * v["match4"] and td <= 0.35 * d["match4"], (step, tv, v["match4"], td, d["match4"])
        f.step(util.DT)


DT = 1.0 / 120.0
CASES = ("sorted", "shuffled", "crowded", "clamped")


def case_inputs(name):
    """Seeded particles: cell-sorted (the tiles take almost every face), the same particles shuffled (mostly the global path), a pile of
    1500 particles in three cells, and particles on the clamp planes and outside the domain."""
    rng = np.random.default_rng({"sorted": 40, "shuffled": 40, "crowded": 41, "clamped": 42}[name])
    dims = (32, 32, 32) if name == "clamped" else (64, 32, 48)
    nx, ny, nz = dims
    n = {"sorted": 120000, "shuffled": 120000, "crowded": 60000, "clamped": 4000}[name]
    pos = np.zeros((n, 4), np.float32)
    if name == "clamped":
        pos[:, :3] = rng.uniform(-3.0, 35.0, (n, 3))
        pos[:50, 0], pos[50:100, 1], pos[100:150, 2] = 31.0, 1.0, 0.5
    else:
        pos[:, 0] = rng.uniform(1.001, nx - 1.001, n)
        pos[:, 1] = rng.uniform(1.001, ny * 0.6, n)
        pos[:, 2] = rng.uniform(1.001, nz - 1.001, n)
    if name == "crowded":
        pos[:1500, 0] = rng.uniform(20.0, 23.0, 1500)
        pos[:1500, 1] = rng.uniform(5.0, 6.0, 1500)
        pos[:1500, 2] = rng.uniform(9.0, 10.0, 1500)
    rows = [rng.normal(0, 3.0, (n, 4)).astype(np.float32) for _ in range(3)]
    c = np.clip(pos[:, :3], 1.0, np.array(dims, np.float32) - 1.0).astype(np.int64)
    order = np.argsort((c[:, 2] * ny + c[:, 1]) * nx + c[:, 0], kind="stable")
    if name == "shuffled":
        order = rng.permutation(n)
    return dims, pos[order], [r[order] for r in rows]


def scatter_hashes(name):
    """SHA-256 of the three velocity taps and the marker after stage 0 (P2G scatter) and of the density residual after stage 9."""
    import blub_b200
    from blub_b200 import fluid as F

    dims, pos, rows = case_inputs(name)
    f = blub_b200.HybridFluid(*dims, pos.shape[0])
    f.set_transfer_path(True)
    f.set_gravity_grid([0.0, -981.0, 0.0])
    f.set_particles(pos, *rows)
    f.step_stages(DT, 0, 1)
    taps = {"ux": F.TAP_UX, "uy": F.TAP_UY, "uz": F.TAP_UZ, "marker": F.TAP_MARKER}
    out = {k: hashlib.sha256(f.download_grid(t).tobytes()).hexdigest() for k, t in taps.items()}
    f.step_stages(DT, 8, 10)
    out["residual"] = hashlib.sha256(f.download_grid(F.TAP_RESIDUAL).tobytes()).hexdigest()
    return out


EXPECTED = {
    "sorted": {
        "ux": "37b8b8d6c75200ebfd1b4ec92d87b28a24b39cefd07b50953a04fc6f149a4d91",
        "uy": "8aa8aa12977e190ed49ef41e4f3d66cff89007b22481d118cf9e2810c6d2df4b",
        "uz": "b6a96f6c86a636c952fc8ec5c6fced583d46979e2f0783608ee6617eb974a348",
        "marker": "dd626fd6d3e7ff713720c7aceb3dcace96d57ace358c6f7a6059fd83a1cfdca6",
        "residual": "ad746f2e2c96e6a379420ff5c8860d809d91852a78454242eb81fc502ff44423",
    },
    "shuffled": {
        "ux": "80f9055db45dab7dc83b60afaf4a8959ca1daae373e09c5cd28ccfcc0bdc688b",
        "uy": "cac2a1b5e6a2856b77d9754a2b325f996e726633170538679a07b6bc4815c782",
        "uz": "8311cd14e392717ff1904b1b9644d54cccf87961e032c52c23a242dc58505fdf",
        "marker": "dd626fd6d3e7ff713720c7aceb3dcace96d57ace358c6f7a6059fd83a1cfdca6",
        "residual": "bea2112664f4efb5de7262a780de98233501e20bd2be9ed782495acf8e938d03",
    },
    "crowded": {
        "ux": "3421e05539c4fee3f50275f9e15cb921e5b52ee16f05aedb8edcfbdcd1002868",
        "uy": "cca8113710b7ffd0b7d2063a0e9a5e6f0945d2b0f17805515ca93c896ba08780",
        "uz": "b44237be38f79bdcc93ed51e386655e3f3876b7b9d4fa40edde38498363d8d15",
        "marker": "05a8a6363850b9ea906e12c59de793ed9909392d5abda40f6612d30072e99179",
        "residual": "50512966e18e466b265f590f9956ccc7b2021a7d05ca9327d542cfb9e3bf62a5",
    },
    "clamped": {
        "ux": "88e53d6c62274a45f32460ede9d040031656f6001fa2f1bdfdd48aadf83dc3a3",
        "uy": "69a64b0985d1eda69873799bbd4abce02c2b7ef1e053b42ab4ec4659777a8c6d",
        "uz": "be61fef11b69827d6ca7e70c11666e92289dd3cc3f981ffdb03458806745819e",
        "marker": "591a3bf4ea5f156a8b6e332c1e28a316b105915e7368a48fa8e2aeeb7eee04d6",
        "residual": "0ed53bd5349604db20d92c8ed8dfa11daec7a95e8ceedf851bba17b11075979a",
    },
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_tiled_scatters_give_the_bits_of_the_untiled_scatter(name):
    assert scatter_hashes(name) == EXPECTED[name]
