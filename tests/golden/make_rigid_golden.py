"""Regenerates tests/golden/rigid_ref.npz by RUNNING the reference's rigid-coupled (CPIC) path: update_rigid_page_map
(/root/reference/src/mpm.cpp:1026-1076), rasterize_rigid_boundary and gather_cdf (src/rigid_transfer.cpp) and the block_op_rigid
branches of rasterize_optimized / resample_optimized (src/transfer.cpp:367-463, 706-835), on the reference's own MPM<3> object,
compiled where they lie by `make -C oracle ref` (oracle/transfer_ref.cpp) against the stand-in core — whose RigidBody is an
ASSUMPTION stated in oracle/taichi_stub/taichi/dynamics/rigid_body.h.  Run in the build container:

    python tests/golden/make_rigid_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import pyoracle as O  # noqa: E402
from taichi_mpm_b200 import scenes  # noqa: E402
from tests import common as T  # noqa: E402

VARIANTS = ["kinematic", "dynamic", "two_bodies", "sand_preset"]


def golden_scene(variant, kind=None, vel=0.3):
    """A stirred block cut by a tilted plate (and, for two_bodies, a small free box inside it).  `kind`: the block of another
    material instead, perturbed at its T.KIND_KW strain (T.perturbed_scene's default otherwise) — not a golden scene."""
    res = 32
    dx = 1.0 / res
    if kind is None:
        kind = scenes.MAT_SAND if variant == "sand_preset" else scenes.MAT_JELLY
        scene, st = T.perturbed_scene(kind, res=res, cells=6, seed=3, strain=0.005, vel=vel)
    else:
        scene, st = T.perturbed_scene(kind, res=res, cells=6, seed=3, vel=vel, **T.KIND_KW.get(kind, {}))
    c = st["x"].mean(0)
    rot = scenes.euler_rotation((7.0, 13.0, -5.0))     # generic orientation: no grid node sits on a triangle edge
    plate = dict(tris=scenes.plate_mesh(0.21, 0.19, axis=1), position=c + np.array([0.004, 0.011, -0.003]), rotation=rot,
                 velocity=(0.1, -0.8, 0.05), angular_velocity=(0.3, 0.0, -0.4), frictions=(0.3, 0.5))
    if variant != "kinematic":
        plate.update(inv_mass=1 / 3.0, inv_inertia=np.diag([40.0, 25.0, 40.0]))
    bodies = [plate]
    if variant == "two_bodies":
        bodies.append(dict(tris=scenes.box_mesh((0.05, 0.04, 0.06)), position=c + np.array([0.09, 0.07, 0.02]),
                           rotation=scenes.euler_rotation((20.0, 5.0, 33.0)), velocity=(-0.5, 0.0, 0.2), friction=-1.0,
                           inv_mass=2.0, inv_inertia=np.diag([300.0, 300.0, 300.0])))
    rigid = scenes.make_rigid(bodies, dx, penalty=1e3)
    if variant == "sand_preset":     # colours the particles bring along: half "positive side of body 1", half of a body that is not there
        n = len(st["x"])
        st["states"] = np.zeros(n, np.uint32)
        st["states"][: n // 2] = 0b1000
        st["states"][n // 2:] = 0b110000
    return scene, st, rigid


def sparse(a):
    flat = a.reshape(-1, a.shape[-1]) if a.ndim == 4 else a.reshape(-1)
    idx = np.nonzero(np.abs(flat).max(1) > 0)[0] if flat.ndim == 2 else np.nonzero(flat)[0]
    return idx.astype(np.int32), flat[idx]


def dense(idx, val, shape):
    g = np.zeros((int(np.prod(shape[:3])),) + tuple(shape[3:]), val.dtype)
    g[idx] = val
    return g.reshape(shape)


def main():
    out = {}
    for v in VARIANTS:
        scene, st, rigid = golden_scene(v)
        new, grid_rast, grid_vel, rs, cdf = O.ref_substep_coupled(scene, st, rigid)
        for name in ("x", "v", "F", "b", "ps", "alive", "states", "bnormal", "bdist", "near"):
            out["%s_%s" % (v, name)] = new[name]
        out[v + "_rigid_v"], out[v + "_rigid_w"] = rs["velocity"], rs["angular_velocity"]
        out[v + "_grid_idx"], out[v + "_grid_val"] = sparse(grid_rast)
        out[v + "_gvel_idx"], out[v + "_gvel_val"] = sparse(grid_vel)
        out[v + "_nstate_idx"], out[v + "_nstate_val"] = sparse(cdf["node_state"])
        out[v + "_ndist_idx"], out[v + "_ndist_val"] = sparse(cdf["node_dist"])
    path = os.path.join(HERE, "rigid_ref.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
