"""CPU checks of what tests/test_gpu_zz_mpm2d_bench.py relies on: its 2-D sand classifier (tests/mpm2d_common.sand_case2d)
names the branch the oracle's return map takes, and the regime guards of its reduced collapse are reachable by the fp32
2-D oracle's own run of the same column."""
import numpy as np

from oracle import pyoracle2d as O
from taichi_mpm_b200 import scenes
from tests import mpm2d_common as MC


def test_sand_classifier_agrees_with_the_oracles_return_map():
    """On sampled F, cdg and logJp, in fp64: case 0 sends both singular values to exp(cohesion), case 1 leaves the trial
    F = cdg F to rounding, case 2 moves it onto the cone (neither of the others)."""
    prm = scenes.material_params(scenes.MAT_SAND)
    rng = np.random.default_rng(50)
    counts = np.zeros(3, np.int64)
    for _ in range(900):
        F = np.eye(2) + rng.normal(size=(2, 2)) * 10.0 ** rng.uniform(-4.0, -0.7)
        cdg = np.eye(2) + rng.normal(size=(2, 2)) * 10.0 ** rng.uniform(-6.0, -2.0)
        ps = 0.0 if rng.random() < 0.4 else rng.uniform(-0.02, 0.02)
        Ft = cdg @ F
        case = int(MC.sand_case2d(Ft[None], prm, [ps])[0])
        Fn, psn = O.plasticity2d(scenes.MAT_SAND, prm, cdg, F, ps)
        s = np.linalg.svd(Fn, compute_uv=False)
        moved = np.abs(Fn - Ft).max()
        if case == 0:
            assert np.abs(s - np.exp(prm[3])).max() <= 1e-12, (Ft, ps, s)
        elif case == 1:
            assert moved <= 1e-13 and psn == 0.0, (Ft, ps, Fn)
        else:
            assert moved > 1e-13 and np.abs(s - np.exp(prm[3])).max() > 1e-12 and psn == 0.0, (Ft, ps, Fn)
        counts[case] += 1
    assert (counts >= 50).all(), counts


def test_fp32_oracle_collapse_reaches_the_reduced_guards():
    """bench_2d.py's column at 64^2 after 0.05 s (625 substeps) of the fp32 2-D oracle meets the guards the engine's run of
    the same column must meet: every return-map case, every floor branch, the compaction and the spread."""
    st, dt, scene = MC.bench_column(64)
    S = st
    for _ in range(int(round(0.05 / dt))):
        S = O.substep2d(scene, S, np.float32, want_grids=False)[0]
    alive = S["alive"].astype(bool)
    S = {k: v[alive] for k, v in S.items()}
    ref, grid_rast, _ = O.substep2d(scene, S, np.float64)
    r = MC.regime2d(st, S, ref, grid_rast, scene)
    print("fp32 oracle, 64^2 at 0.05 s", r)
    bad = {k: (r[k], g) for k, g in MC.GUARDS_REDUCED[(64, 0.05)].items() if not r[k] > g}
    assert not bad, bad
