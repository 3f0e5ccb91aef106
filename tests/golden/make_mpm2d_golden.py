"""Regenerates tests/golden/mpm2d_ref.npz and tests/golden/frame2d_ref.bgeo by RUNNING the reference's 2-D solver MPM<2>
(/root/reference/src/mpm.cpp, transfer.cpp — the scalar rasterize / resample MPM<2> runs —, particles.cpp at dim = 2,
visualize.cpp) compiled where it lies by oracle/pyoracle2d.ref_build() (oracle/transfer2d_ref.cpp, reft2_*; stand-in core headers
oracle/taichi_stub/taichi/*.h, vendored SPGrid and Partio).  Per material:
  * one substep stage by stage: the node (momentum, mass) after P2G, the node velocities after the grid update, the
    particles after G2P and clear_boundary_particles;
  * SUBSTEPS whole substeps by MPM<2>::substep() itself, with two particles placed in the 7-cell deletion band;
and one frame of MPM<2>::write_partio after three substeps of the sand scene.  Run in the build container:

    python tests/golden/make_mpm2d_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import pyoracle2d as O  # noqa: E402
from tests.mpm2d_common import scene2d  # noqa: E402

KINDS = [0, 1, 2, 3, 4, 5, 6, 7]
SUBSTEPS = 12
FRAME_SUBSTEPS = 3
# per-kind scene arguments: von Mises at a strain that puts particles on both sides of its yield surface, visco hardening
KIND_KW = {6: dict(strain=0.006), 7: dict(kappa=0.3)}


def golden_scene(kind):
    """A 32^2 grid, an 8 x 8-cell block (256 particles) stirred by a random affine velocity field over a floor plane with
    Coulomb friction 0.4."""
    return scene2d(kind, seed=30 + kind, **KIND_KW.get(kind, {}))


def substep_scene(kind):
    """The same block with two particles moved into the 7-cell band (src/mpm.h:269-276): the first substep deletes them."""
    scene, st = golden_scene(kind)
    st["x"][0] = [6.5 / 32, 0.5]
    st["x"][1] = [0.5, (32 - 6.5) / 32]
    return scene, st


def sparse(grid):
    flat = grid.reshape(-1, 4)
    idx = np.nonzero(np.abs(flat).max(1) > 0)[0].astype(np.int32)
    return idx, flat[idx]


def dense(idx, val, res=(32, 32)):
    g = np.zeros(((res[0] + 1) * (res[1] + 1), 4), np.float32)
    g[idx] = val
    return g.reshape(res[0] + 1, res[1] + 1, 4)


def reference_run(kind):
    """What the reference computes for `kind`: a dict of the fixture's arrays for that kind."""
    out = {}
    scene, st = golden_scene(kind)
    r = O.RefSolver2D(scene, st)
    r.stage(1)
    out["grid_rast"] = sparse(r.get_grid())
    r.stage(2)
    out["grid_vel"] = sparse(r.get_grid())
    r.stage(3)
    out["stage"] = r.particles()
    r.close()
    scene, st = substep_scene(kind)
    r = O.RefSolver2D(scene, st)
    r.substep(SUBSTEPS)
    out["sub"] = r.particles()
    r.close()
    flat = {}
    for k in ("grid_rast", "grid_vel"):
        flat["k%d_%s_idx" % (kind, k)], flat["k%d_%s_val" % (kind, k)] = out[k]
    for tag in ("stage", "sub"):
        for k, a in out[tag].items():
            flat["k%d_%s_%s" % (kind, tag, k)] = a
    return flat


def write_frame(path):
    scene, st = golden_scene(4)
    r = O.RefSolver2D(scene, st)
    r.substep(FRAME_SUBSTEPS)
    r.write_partio(path)
    r.close()


def main():
    out = {}
    for kind in KINDS:
        out.update(reference_run(kind))
    path = os.path.join(HERE, "mpm2d_ref.npz")
    np.savez_compressed(path, **out)
    write_frame(os.path.join(HERE, "frame2d_ref.bgeo"))
    print("wrote", path, "and frame2d_ref.bgeo")


if __name__ == "__main__":
    main()
