"""A 2-D sand column collapsing on a floor with a circular obstacle (MPM<2>), written as BGEO frames:

    python examples/sand_column_2d.py [frames] [res] [frame_directory]

MPM2D(res=(r, r)) builds the 2-D engine; add_particles(benchmark_block=...) seeds 4 particles per cell.  Half-way a second,
smaller column of snow is dropped in: the sand keeps its ids.  Each frame prints the particle count and how far the column has
spread.  (The reference's scripts/mls-cpic/sand_wheel_2D.py also needs a 2-D rigid wheel, which the engine does not have.)"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from taichi_mpm_b200 import MPM2D  # noqa: E402


def main(frames=4, res=64, frame_directory=None):
    frame_directory = frame_directory or tempfile.mkdtemp(prefix="sand2d_")
    mpm = MPM2D(res=(res, res), base_delta_t=2e-5 * 256 / res, frame_dt=2e-3, frame_directory=frame_directory)
    ls = mpm.create_levelset()
    ls.add_plane((0, 1), -8.0 / res)                 # the floor, 8 cells up
    ls.add_sphere((0.7, 0.2), 0.06)                  # an obstacle in the column's way
    ls.set_friction(0.4)
    mpm.set_levelset(ls)
    c0, c1 = res // 4, res // 2
    mpm.add_particles(type="sand", benchmark_block=((c0, 8), (c1, 8 + res // 3)), density=400)
    sand = mpm.get_particles()["id"]
    for f in range(frames):
        if f == frames // 2:
            before = mpm.get_particles()
            mpm.add_particles(type="snow", benchmark_block=((c1 + 4, res // 2), (c1 + 8, res // 2 + 4)), initial_velocity=(0.0, -1.0))
            after = mpm.get_particles()
            assert np.array_equal(after["id"][: len(before["id"])], before["id"]), "ids changed"
            assert np.array_equal(after["x"][: len(before["id"])], before["x"]), "state changed"
        mpm.step(mpm.frame_dt)
        fn = mpm.visualize()
        p = mpm.get_particles()
        print("frame %d: %d particles, sand spans x in [%.3f, %.3f], %s" % (f + 1, len(p["id"]), p["x"][: len(sand), 0].min(),
                                                                          p["x"][: len(sand), 0].max(), os.path.basename(fn)))
    return mpm


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]), *(sys.argv[3:4]))
