"""Writes the scene fixtures used by the tests and by bench.py.

The scene PARAMETERS of the reference's shipped scenes are restated here (cited) and emitted as blub scene JSON (same schema as
src/scene/mod.rs:19-43); `tests/test_host.py` checks them against the reference's scene files, stored unchanged under
tests/golden/reference_scenes.  The synthetic scenes are the ones SURVEY.md section 0.1 /
BASELINE.json ask for (256^3 with ~16M particles, 512^3 with ~64M).

    python tests/golden/make_scenes.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def scene(dim, scale, max_particles, cubes, gravity=(0.0, -9.81, 0.0)):
    v = lambda t: {"x": t[0], "y": t[1], "z": t[2]}
    return {
        "gravity": v(gravity),
        "fluid": {
            "world_position": v((0.0, 0.0, 0.0)),
            "max_num_particles": max_particles,
            "grid_to_world_scale": scale,
            "grid_dimension": v(dim),
            "fluid_cubes": [{"min": v(a), "max": v(b)} for a, b in cubes],
        },
    }


SCENES = {
    # scenes/single_cell_debug.json:13-31 -- 8 particles in one cell of a 64x64x128 grid (config C1)
    "single_cell_debug": scene((64, 64, 128), 0.01, 1238328, [((0.319, 0.319, 0.639), (0.32, 0.32, 0.64))]),
    # scenes/dam_halfhalf.json:13-31 -- 128x64x64, 1,218,672 particles (config C2)
    "dam_halfhalf": scene((128, 64, 64), 0.01, 1238328, [((0.0, 0.0, 0.0), (0.64, 0.4, 0.64))]),
    # scenes/dam_halfhalf_highres.json:13-31 -- 256x128x128, 10,113,264 particles (config C3)
    "dam_halfhalf_highres": scene((256, 128, 128), 0.005, 10193528, [((0.0, 0.0, 0.0), (0.64, 0.4, 0.64))]),
    # scenes/filled_basin.json:13-31 -- 64^3 basin
    "filled_basin": scene((64, 64, 64), 0.01, 1238328, [((0.0, 0.0, 0.0), (0.64, 0.32, 0.64))]),
    # synthetic C3': 256^3 grid, cube [1,128)^3 -> 127^3 * 8 = 16,387,064 particles (SURVEY.md section 0.1)
    "dam_256": scene((256, 256, 256), 0.005, 16500000, [((0.0, 0.0, 0.0), (0.64, 0.64, 0.64))]),
    # synthetic C4: 512^3 basin, 510 x 31 x 510 cells -> 64,504,800 particles
    "basin_512": scene((512, 512, 512), 0.01, 65000000, [((0.0, 0.0, 0.0), (5.12, 0.32, 5.12))]),
    # scenes/double_dam_wgpulogo.json:13-40 without its static object -- 128x64x64, two dams, 1,199,328 particles (config C5's fluid)
    "double_dam": scene((128, 64, 64), 0.01, 2000000, [((0.0, 0.0, 0.0), (0.32, 0.4, 0.64)), ((0.96, 0.0, 0.0), (1.28, 0.4, 0.64))]),
    # small dam break for per-stage parity (not a reference scene)
    "dam_small": scene((32, 32, 32), 0.01, 40000, [((0.0, 0.0, 0.0), (0.16, 0.2, 0.32))]),
}

if __name__ == "__main__":
    out = os.path.join(HERE, "scenes")
    os.makedirs(out, exist_ok=True)
    for name, sc in SCENES.items():
        with open(os.path.join(out, name + ".json"), "w") as fh:
            json.dump(sc, fh, indent=1)
            fh.write("\n")
    print("wrote", len(SCENES), "scenes to", out)
