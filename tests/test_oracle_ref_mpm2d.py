"""Pin of the oracle's 2-D substep (oracle_substep2d, pyoracle2d.substep2d) against the REFERENCE's own MPM<2>: src/mpm.cpp,
transfer.cpp (the scalar rasterize / resample MPM<2> runs), particles.cpp at dim = 2 and the vendored SPGrid, compiled where
they lie (oracle/transfer2d_ref.cpp, reft2_*).  Stage by stage — the node (momentum, mass) after P2G, the node velocities after
the grid update, the particles after G2P and deletion — and as whole substeps by MPM<2>::substep() itself, for all eight
materials: the same survivors, the trajectories at the tolerances of the 3-D pins (tests/test_oracle_ref_transfer.py).  Golden
vectors of the reference's run are committed (tests/golden/mpm2d_ref.npz); where the reference tree is present the same runs
happen live, together with the level-set modes, clean_boundary 0, particles in the band and the dampings."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import pyoracle2d as O
from taichi_mpm_b200 import scenes
from tests import common as T
from tests.mpm2d_common import scene2d

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_mpm2d_golden", os.path.join(HERE, "golden", "make_mpm2d_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

# the 3-D pins' bounds: one stage (TOL) and whole substeps (TOL_SUB); visco_tau relative (the reference forms |P| - tau in fp32)
TOL = dict(grid=3e-6, x=2e-7, v=3e-6, F=2e-6, b=4e-5, ps=1e-5)
TOL_SUB = dict(x=2e-6, v=1e-5, F=1.5e-5, b=2e-4, ps=1.5e-5)
LIVE = pytest.mark.skipif(not O.ref_available(), reason="reference tree absent: golden vectors only")


def _golden():
    return np.load(os.path.join(HERE, "golden", "mpm2d_ref.npz"))


def _assert_particles(ref, new, alive, tol, kind):
    s = alive.astype(bool)
    assert np.abs(ref["x"][s] - new["x"][s]).max() <= tol["x"]
    assert np.abs(ref["v"][s] - new["v"][s]).max() <= tol["v"] * np.abs(new["v"][s]).max()
    assert np.abs(ref["b"][s] - new["b"][s]).max() <= tol["b"] * np.abs(new["b"][s]).max()
    if kind != scenes.MAT_WATER:   # water carries no F
        assert np.abs(ref["F"][s] - new["F"][s]).max() <= tol["F"]
    assert T.ps_err(ref["ps"][s], new["ps"][s]) <= (5e-4 if kind == scenes.MAT_VISCO and tol is TOL_SUB else tol["ps"])


def _assert_stages(kind, grid_rast_ref, grid_vel_ref, p_ref):
    scene, st = G.golden_scene(kind)
    new, grid_rast, grid_vel = O.substep2d(scene, st, np.float64)
    pmax = max(np.abs(grid_rast[..., :2]).max(), grid_rast[..., 3].max())
    assert np.abs(grid_rast_ref - grid_rast).max() <= TOL["grid"] * pmax
    assert ((grid_rast_ref[..., 3] > 0) == (grid_rast[..., 3] > 0)).all()            # the same nodes touched
    act = grid_rast[..., 3] > 0
    assert np.abs(grid_vel_ref[..., :2] - grid_vel[..., :2])[act].max() <= 5e-6 * np.abs(grid_vel[..., :2]).max()
    assert np.array_equal(p_ref["alive"], new["alive"])
    _assert_particles(p_ref, new, new["alive"], TOL, kind)


def _assert_substeps(kind, scene, st, p_ref, n):
    cur = dict(st)
    for _ in range(n):
        cur = O.substep2d(scene, cur, np.float64, want_grids=False)[0]
    assert np.array_equal(p_ref["alive"], cur["alive"])                            # the same particles were deleted
    _assert_particles(p_ref, cur, cur["alive"], TOL_SUB, kind)
    return cur


@pytest.mark.parametrize("kind", G.KINDS)
def test_oracle_stages_match_golden_run_of_reference(kind):
    z = _golden()
    p_ref = {k: z["k%d_stage_%s" % (kind, k)] for k in ("x", "v", "F", "b", "ps", "alive")}
    _assert_stages(kind, G.dense(z["k%d_grid_rast_idx" % kind], z["k%d_grid_rast_val" % kind]),
                   G.dense(z["k%d_grid_vel_idx" % kind], z["k%d_grid_vel_val" % kind]), p_ref)


@pytest.mark.parametrize("kind", G.KINDS)
def test_oracle_substeps_match_golden_run_of_reference_substep(kind):
    z = _golden()
    p_ref = {k: z["k%d_sub_%s" % (kind, k)] for k in ("x", "v", "F", "b", "ps", "alive")}
    scene, st = G.substep_scene(kind)
    cur = _assert_substeps(kind, scene, st, p_ref, G.SUBSTEPS)
    assert not cur["alive"][:2].any() and cur["alive"][2:].all()                   # the two band particles, and only they


@pytest.mark.parametrize("kind", G.KINDS)
def test_fp64_and_fp32_oracle_agree_to_fp32_rounding(kind):
    scene, st = G.golden_scene(kind)
    a, ga, _ = O.substep2d(scene, st, np.float64)
    b, gb, _ = O.substep2d(scene, st, np.float32)
    assert np.array_equal(a["alive"], b["alive"])
    assert np.abs(ga - gb).max() <= 2e-6 * np.abs(ga).max()
    _assert_particles(b, a, a["alive"], TOL, kind)


@LIVE
def test_golden_is_what_the_reference_computes():
    z = _golden()
    for kind in G.KINDS:
        fresh = G.reference_run(kind)
        for k, a in fresh.items():
            assert z[k].shape == np.shape(a) and np.abs(z[k].astype(np.float64) - np.asarray(a, np.float64)).max(initial=0) <= 1e-6, k


@LIVE
@pytest.mark.parametrize("friction", [-1.0, -2.0, 0.4])
@pytest.mark.parametrize("clean", [1, 0])
def test_level_set_modes_and_the_band_match_reference_substeps_live(friction, clean):
    """A block sliding into a tilted floor and towards the band, 15 substeps by MPM<2>::substep() itself.  (No node lies on a
    plane, on the -3 cut-off or where the two planes tie: the stand-in level set and scenes.planes_sdf2d round phi in different
    orders.)"""
    res = 32
    scene, st = scene2d(scenes.MAT_JELLY, res=(res, res), blocks=[((4, 9), (12, 15))], clean_boundary=clean, friction=friction, seed=40,
                        levelset=("planes", [[0.0, 1.0, 0.0, -8.6], [0.6, 0.8, 0.0, -13.1]]), vel=0.3)
    st["v"][:, 0] -= 6.0 if clean else 60.0   # towards the x = 0 face
    st["x"][0] = [6.8 / res, 12.0 / res]     # in the band from the start
    r = O.RefSolver2D(scene, st)
    r.substep(15)
    p_ref = r.particles()
    cur = _assert_substeps(scenes.MAT_JELLY, scene, st, p_ref, 15)
    if clean:
        assert 0 < cur["alive"].sum() < len(st["x"])
    else:   # without the band the block runs on towards the face
        assert (cur["x"][:, 0] * res < 3.0).any()


@LIVE
@pytest.mark.parametrize("apic,rpic", [(0.4, 0.0), (0.0, 0.6), (0.3, 0.2)])
def test_dampings_match_reference_substeps_live(apic, rpic):
    scene, st = scene2d(scenes.MAT_SNOW, seed=41, apic=apic, rpic=rpic)
    r = O.RefSolver2D(scene, st)
    r.substep(10)
    _assert_substeps(scenes.MAT_SNOW, scene, st, r.particles(), 10)


@LIVE
@pytest.mark.parametrize("kind", [scenes.MAT_SAND, scenes.MAT_WATER, scenes.MAT_VISCO])
def test_longer_runs_match_reference_substeps_live(kind):
    """25 substeps, grid gravity (particle_gravity = 0) with a sideways component."""
    scene, st = scene2d(kind, seed=42, particle_gravity=0, gravity=(2.0, -9.0), **G.KIND_KW.get(kind, {}))
    r = O.RefSolver2D(scene, st)
    r.substep(25)
    _assert_substeps(kind, scene, st, r.particles(), 25)
