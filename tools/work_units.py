"""Which work unit should the sparse PCG kernel hand out?  For marker volumes of a dam break (here: generated with the CPU oracle,
tools have no GPU), count for several unit shapes how many units hold fluid, how many sequential passes a persistent grid of
BLOCKS blocks x 8 warps needs per phase, and how full the processed units are.

    python tools/work_units.py markers.npz        # arrays m<step> of shape [nz, ny, nx], FLUID = 1
"""
import sys

import numpy as np

BLOCKS = 132 * 3  # the column solver's grid on an H100 SXM: three resident blocks on each of 132 SMs
SHAPES = [("tile 128x8x4 / block", (128, 8, 4), BLOCKS), ("brick 32x8x4 / 2 warps", (32, 8, 4), BLOCKS * 4), ("brick 32x4x4 / warp", (32, 4, 4), BLOCKS * 8),
          ("brick 64x2x4 / warp", (64, 2, 4), BLOCKS * 8), ("brick 128x1x4 / warp (row)", (128, 1, 4), BLOCKS * 8), ("brick 16x8x4 / warp", (16, 8, 4), BLOCKS * 8)]


def main(path):
    data = np.load(path)
    for key in sorted(data.files, key=lambda k: int(k[1:])):
        fl = data[key] == 1
        nz, ny, nx = fl.shape
        cols = fl.reshape(nz // 4, 4, ny, nx // 4, 4).any(axis=4)  # [tz, plane, y, quad]: the (thread, plane) units of the kernel
        print(f"step {key[1:]}: {100 * fl.mean():.1f} % of the cells FLUID, {100 * cols.mean():.1f} % of the (quad, plane) units")
        for name, (bx, by, bz), workers in SHAPES:
            if nx % bx or ny % by or nz % bz:
                continue
            act = fl.reshape(nz // bz, bz, ny // by, by, nx // bx, bx).any(axis=(1, 3, 5))
            n_act = int(act.sum())
            # fill of the processed units: fluid-holding (quad, plane) units / all (quad, plane) units of the active work units
            u = cols.reshape(nz // 4, 4, ny // by, by, nx // bx, bx // 4).sum(axis=(1, 3, 5))
            fill = u[act.reshape(u.shape)].sum() / max(1, n_act * (bx // 4) * by * 4)
            print(f"    {name:28s} active {100 * act.mean():5.1f} %  = {n_act:6d} units, {int(np.ceil(n_act / workers)):3d} pass(es) of {workers} workers"
                  f" (ideal {n_act / workers:5.2f}), fill {100 * fill:5.1f} %")


if __name__ == "__main__":
    main(sys.argv[1])
