"""The engine's own kernels on the edge states of tests/material_states.py: rotated, large, degenerate, near-singular
and inverted deformation gradients, every kind, one particle per tile (as test_gpu_next_p2g.py::_probe_state) so that
each particle's affine matrix can be recovered from the next P2G.  One substep against the fp64 oracle (grid, x, v, b,
F, ps), then the next P2G: k_refresh_affine's A at upload and k_g2p's cache after the substep."""
import numpy as np
import pytest

from oracle import pyoracle as O
from taichi_mpm_b200 import scenes
from tests import common as T
from tests import material_states as MS
from tests.test_gpu_next_p2g import PROBE_DT, PROBE_RES, PROBE_SLOTS, PROBE_TOL_A, TOL_STRESS, _math, _recover_affine

pytestmark = pytest.mark.gpu

# per kind and regime, on the device
PER_REGIME = 12


def edge_particles(kind):
    """F and ps of the edge regimes where the reference's step is defined at upload and after it: the oracle's
    calculate_force of the uploaded F must be finite (the Hencky stress of an inverted F is log of a negative sigma, and
    so is visco's return map), and near-singular states keep s_min >= 1e-2 (test_host_math.py::edge_errors)"""
    prm = scenes.material_params(kind)
    Fs, pss = [], []
    for regime in MS.REGIMES:
        if regime == "near_singular" and kind in (scenes.MAT_VON_MISES, scenes.MAT_VISCO):
            continue   # their return maps scale F by s'/s_min with s_min from e = s^2 - 1: test_gpu_device_math.py checks det F'
        for strain in (MS.ROTATED_STRAIN[kind] if regime == "rotated" else (None,)):
            F, _, ps, _ = MS.states(kind, regime, 4 * PER_REGIME, 5, strain)
            ok = MS.min_abs_sigma(F) >= 5e-3
            if kind in MS.HENCKY + (scenes.MAT_VISCO,):
                ok &= np.linalg.det(F.astype(np.float64)) > 0
            ok &= np.array([np.isfinite(O.calculate_force(kind, prm, F[i].astype(np.float64), float(ps[i]), 1.0)).all() for i in range(len(F))])
            Fs.append(F[ok][:PER_REGIME]); pss.append(ps[ok][:PER_REGIME])
    return np.concatenate(Fs), np.concatenate(pss)


def edge_scene(kind, particle_gravity, seed=7):
    rng = np.random.default_rng(seed + kind)
    F, ps = edge_particles(kind)
    n = len(F)
    dx = 1.0 / PROBE_RES
    ks = np.stack(np.meshgrid(*[np.arange(2, 2 + PROBE_SLOTS)] * 3, indexing="ij"), -1).reshape(-1, 3)
    ks = ks[rng.permutation(len(ks))][:n]
    assert len(ks) == n
    X = 4 * ks + 1 + rng.uniform(0.6, 1.4, (n, 3))
    vol = np.full(n, dx ** 3 / 8, np.float32)
    st = scenes.make_state((X * dx).astype(np.float32), (vol * 400).astype(np.float32), vol, kind)
    st["F"] = np.ascontiguousarray(F.transpose(0, 2, 1).reshape(n, 9), np.float32)
    st["ps"] = ps.astype(np.float32)
    st["group"] = np.zeros(n, np.int32)
    st["v"] = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32)
    st["b"] = np.ascontiguousarray((rng.normal(size=(n, 3, 3)) * 1e-3).transpose(0, 2, 1).reshape(n, 9), np.float32)
    scene = dict(res=(PROBE_RES,) * 3, dx=dx, dt=PROBE_DT, gravity=(0.0, -10.0, 0.0), particle_gravity=particle_gravity,
                 mat_kind=np.array([kind], np.int32), mat_params=np.array([scenes.material_params(kind)], np.float32), planes=None,
                 friction=0.0, sdf=None)
    return scene, st


def affine_error(e, scene):
    """A recovered from the engine's next P2G against A of the oracle's calculate_force of the downloaded state, per
    particle relative to its own stress term plus 1e-2 of the batch's largest (test_gpu_next_p2g.py::_probe)"""
    S = e.download()
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g = e.download_grid(0).astype(np.float64)
    e.resample()
    A = _recover_affine(g, S, scene["dx"])
    S_ = -4.0 / float(np.float32(scene["dx"])) * scene["dt"]
    Fm, bm = _math(S["F"]), _math(S["b"])
    kind, prm = int(scene["mat_kind"][0]), scene["mat_params"][0]
    stress = np.stack([O.calculate_force(kind, prm, Fm[i], float(S["ps"][i]), float(S["vol"][i])) * S_ for i in range(len(Fm))])
    ref = stress + 4.0 * S["mass"].astype(np.float64)[:, None, None] * bm
    scale = np.abs(stress).max((1, 2)) + 1e-2 * np.abs(stress).max()
    return float((np.abs(A - ref).max((1, 2)) / scale).max())


KINDS = [("linear", scenes.MAT_LINEAR), ("jelly", scenes.MAT_JELLY), ("snow", scenes.MAT_SNOW), ("water", scenes.MAT_WATER),
         ("sand", scenes.MAT_SAND), ("elastic", scenes.MAT_ELASTIC), ("von_mises", scenes.MAT_VON_MISES), ("visco", scenes.MAT_VISCO)]


@pytest.mark.parametrize("particle_gravity", [0, 1], ids=["grid_gravity", "particle_gravity"])
@pytest.mark.parametrize("name,kind", KINDS)
def test_edge_states_substep_and_next_p2g(name, kind, particle_gravity):
    scene, st = edge_scene(kind, particle_gravity)
    e = T.make_engine(scene, st)
    a0 = affine_error(e, scene)                       # the A of the upload (k_refresh_affine); resample advanced the state
    e.close()
    e = T.make_engine(scene, st)
    err, got, ref = T.compare_substep(e, scene, st)
    a1 = affine_error(e, scene)                       # k_g2p's cache of the substep above
    e.close()
    print(name, "pg=%d" % particle_gravity, "n=%d" % len(st["x"]), {k: "%.3g" % v for k, v in err.items() if not isinstance(v, bool)},
          "A upload %.3g A g2p %.3g" % (a0, a1))
    assert err["alive_match"], err
    # slow isolated particles: the stress is most of each node's momentum and of v and b after one substep, so those
    # take the next-P2G tolerance relative to the stress (TOL_STRESS); the per-state stress errors behind them are
    # bounded in test_gpu_device_math.py (2e-4 of the scale, or 2x the reference's own fp32 error for rotated states:
    # a 1e-4 sand strain under a half turn is resolved to ~5e-4 in fp32)
    assert err["grid_rast"] <= TOL_STRESS and err["grid_vel"] <= TOL_STRESS, err
    assert err["x"] <= T.TOL_X_ABS and err["v"] <= TOL_STRESS and err["b"] <= TOL_STRESS, err
    # F per particle relative to max(1, |F'|) (stretches up to 5), as test_host_math.py::edge_errors
    Fr = ref["F"][got["id"].astype(np.int64)]
    F_rel = float((np.abs(got["F"] - Fr).max(1) / np.maximum(1.0, np.abs(Fr).max(1))).max())
    assert F_rel <= T.TOL_F_ABS and err["ps"] <= T.TOL_PS_ABS, (F_rel, err)
    assert a0 <= PROBE_TOL_A and a1 <= PROBE_TOL_A, (a0, a1)
