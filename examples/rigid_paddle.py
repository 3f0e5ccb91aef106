"""A scripted paddle pushed through a sand pile, the way the reference's CPIC scripts set scenes up
(scripts/mls-cpic/sand_stir.py:43-51, sand_sweep.py), on the mirror + device engine:

    python examples/rigid_paddle.py [frames] [res]

The colour field, gather_cdf, the coupled transfers and the paddle's advance run on the device, a whole frame per engine call;
the paddle's motion is a Python callable (where the reference wraps one in tc.function13), evaluated on the host once per frame
into the table of poses the device follows."""
import sys

import numpy as np

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from taichi_mpm_b200 import MPM, scenes  # noqa: E402


def main(frames=2, res=48):
    mpm = MPM(res=(res, res, res), base_delta_t=1e-4, frame_dt=2e-3, penalty=1e3)
    ls = mpm.create_levelset()
    ls.add_plane((0, 1, 0), -0.2)
    ls.set_friction(0.4)
    mpm.set_levelset(ls, False)
    lo, hi = int(0.3 * res), int(0.7 * res)
    mpm.add_particles(type="sand", benchmark_block=((lo, int(0.2 * res) + 1, lo), (hi, int(0.45 * res), hi)), density=400.0, jitter=0.2)
    mpm.add_particles(type="rigid", tris=scenes.plate_mesh(0.02, 0.15, axis=0), codimensional=True, friction=0.3,
                      scripted_position=lambda t: (0.35 + 0.8 * t, 0.33, 0.5), scripted_rotation=lambda t: (0.0, 0.0, 10.0))
    x0 = mpm.get_particles()["x"].mean(0)
    for f in range(frames):
        mpm.step(mpm.frame_dt)
        p = mpm.get_particles()
        pc = mpm.engine.get_particle_cdf(mpm._n_uploaded)
        print("frame %d: t=%.4f  %d particles, %d coloured, %d near the paddle, centre of mass moved %s" %
              (f + 1, float(mpm.get_current_time()), len(p["x"]), int((pc["states"] != 0).sum()), int(pc["near"].sum()), np.round(p["x"].mean(0) - x0, 5)))
    return mpm


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
