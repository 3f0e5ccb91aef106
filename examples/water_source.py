"""A water jet into a container, the shape of scripts/async/water.py: every frame `frame_update` adds a slab of water at the
inlet (MPM.add_particles mid-run), which the engine appends to the resident set on the device:

    python examples/water_source.py [frames] [res]

Each frame prints the particle count and checks that the particles of earlier frames kept their ids (the BGEO `index`
attribute a tool follows particles by)."""
import sys

import numpy as np

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from taichi_mpm_b200 import MPM  # noqa: E402


def main(frames=4, res=32):
    dx = 1.0 / res
    mpm = MPM(res=(res, res, res), base_delta_t=1e-4, frame_dt=2e-3, gravity=(0.0, -1.0, 0.0))
    ls = mpm.create_levelset()
    ls.add_cuboid((0.25, 0.25, 0.25), (0.75, 0.75, 0.75), inside_out=True)      # the container: everything outside is solid
    ls.set_friction(0.0)
    mpm.set_levelset(ls)
    # the inlet: a 2-cell-thick slab of 4 x 4 cells near the container's left wall, 8 particles per cell
    c = np.stack(np.meshgrid(np.arange(2), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(-1, 3)
    lattice = np.array([[i, j, k] for i in (0.25, 0.75) for j in (0.25, 0.75) for k in (0.25, 0.75)])
    slab = ((c[:, None, :] + lattice[None]).reshape(-1, 3) * dx + np.array([0.3, 0.55, 0.45])).astype(np.float32)
    state = {}

    def frame_update(t, frame_dt):
        if mpm.num_particles() > 0:
            p = mpm.get_particles()
            state["ids"], state["x"] = p["id"], p["x"]
        mpm.add_particles(type="water", positions=slab, initial_velocity=(2.0, 0.0, 0.0))
        if "ids" in state:
            q = mpm.get_particles()
            old = np.isin(q["id"], state["ids"])
            assert np.array_equal(q["id"][old], state["ids"]) and np.array_equal(q["x"][old], state["x"]), "earlier ids changed"
            assert q["id"][~old].min() > state["ids"].max(), "new ids do not follow the earlier ones"

    for f in range(frames):
        frame_update(float(mpm.get_current_time()), mpm.frame_dt)
        mpm.step(mpm.frame_dt)
        print("frame %d: %d particles, ids 0..%d, earlier ids unchanged" % (f + 1, mpm.num_particles(), mpm.get_particles()["id"].max()))
    return mpm


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
