"""The 2-D engine where bench_2d.py runs it, against the fp64 2-D oracle: the full-size columns at rest and in the developed
collapse, the same collapse at reduced size further on, and large and non-square grids.

bench_2d.py times its sand column at 1024^2 (1.05 M particles) and 2048^2 (4.19 M) at rest and after 0.05 s of collapse.
There the column is compacted at its floor (6 to 8 particles per cell), its floor nodes stick, slide and separate, its sand
sits in every case of the return map, and the sort keys run at 21 and 23 bits, with the dead-row key res0 res1 exactly
2^20 and 2^22.  The tests reach each state on the engine's own path (one upload, then e.substep(n), graph-replayed) and
check it:

- test_bench_state_full_size: bench_2d's columns at its two sizes, at rest (substep 20) and developed (substep 10 440 at
  1024^2, 20 440 at 2048^2): one substep stage by stage against the fp64 oracle on every particle and node; the regime
  guards at the developed state.
- test_full_size_invariants: the first P2G's mass and momentum, ids, mass and vol after the developed run, two engines
  bit-identical, host launches bit-identical to graph replay from the developed state.
- test_reduced_developed_collapse: the column at res / 2 cells on 64^2 to 256^2 grids after 0.05 s and 0.3 s (band
  deletions by then), three chained substeps; 64^2 also runs on the SIMT emulator (tests/test_mpm2d_simt.py).
- test_large_grids: 2^20 and 2^22 cells, a non-square 2^22, and two grids whose dx is not a power of two, with blocks
  dying in the band and at the faces in the same substep, and a block in the last node tile; two chained substeps.

Bounds: tests/test_gpu_mpm2d.assert_parity_yardstick, the tests/common.py bound of each metric or, for the grid, the
velocity-normalised metrics, F and ps, 4x the fp32 oracle's own error on the same substep; x keeps its common bound, mass
is exact.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit, card read in the same run), engine error / fp32 yardstick, worst
over the case's checked substeps (common bounds: grid 2e-5, v and b 1e-4, F 2e-5, ps 1e-5; x was <= 1.6e-7 everywhere):

| case | grid_rast | grid_vel | grid_vel_heavy | v | b | F | ps |
|---|---|---|---|---|---|---|---|
| 1024^2 at rest (20) | 2.1e-7 / 2.4e-7 | 3.6e-7 / 1.9e-3 | 3.6e-7 / 1.9e-3 | 3.2e-7 / 3.1e-4 | 1.2e-6 / 1.9e-3 | 2.0e-7 / 2.3e-7 | 5.6e-9 / 5.6e-9 |
| 1024^2 developed (10 440) | 4.2e-7 / 3.9e-7 | 7.9e-7 / 7.6e-6 | 7.9e-7 / 5.8e-6 | 4.2e-7 / 1.1e-6 | 8.8e-6 / 2.3e-5 | 3.4e-7 / 4.0e-7 | 3.9e-7 / 3.9e-7 |
| 2048^2 at rest (20) | 2.9e-7 / 2.6e-7 | 5.3e-7 / 3.8e-3 | 5.3e-7 / 3.8e-3 | 3.1e-7 / 5.7e-4 | 1.5e-6 / 4.0e-3 | 1.5e-7 / 2.2e-7 | 2.5e-9 / 2.5e-9 |
| 2048^2 developed (20 440) | 3.8e-7 / 4.0e-7 | 0.663 / 0.663 (*) | 1.7e-6 / 5.1e-6 | 4.5e-7 / 1.1e-6 | 1.3e-5 / 2.8e-5 | 3.3e-7 / 3.9e-7 | 3.6e-7 / 3.6e-7 |
| reduced, 64^2 to 256^2, 0.05 s | 4.2e-7 / 4.5e-7 | 1.3e-6 / 7.5e-6 | 5.5e-7 / 6.7e-6 | 4.3e-7 / 1.2e-6 | 6.5e-6 / 1.9e-5 | 3.9e-7 / 4.2e-7 | 3.5e-7 / 3.5e-7 |
| reduced, 128^2 and 256^2, 0.3 s | 3.3e-7 / 4.0e-7 | 0.303 / 0.303 (*) | 1.8e-6 / 2.0e-6 | 4.0e-7 / 5.0e-7 | 7.4e-6 / 8.3e-6 | 4.0e-7 / 3.8e-7 | 3.5e-7 / 3.5e-7 |
| power-of-two large grids | 2.3e-7 / 4.3e-7 | 4.4e-6 / 4.4e-6 | <= 4.4e-6 | 3.9e-7 / 5.5e-7 | 2.4e-5 / 2.3e-5 | 5.3e-6 / 5.6e-6 | 1.7e-6 / 2.9e-6 |
| 2047 x 2050, dx = 0.9 / 2047 | 7.2e-5 / 7.2e-5 | 1.2e-4 / 1.2e-4 | 1.2e-4 / 1.2e-4 | 2.3e-5 / 2.3e-5 | 3.4e-4 / 3.4e-4 | 6.1e-5 / 6.1e-5 | 2.3e-5 / 2.3e-5 |
| 1000 x 1536, dx = 1 / 1000 | 3.0e-5 / 3.0e-5 | 1.9e-5 / 1.9e-5 | 1.9e-5 / 1.9e-5 | 1.0e-6 / 1.0e-6 | 1.5e-4 / 1.6e-4 | 3.7e-6 / 3.7e-6 | 3.5e-6 / 3.5e-6 |

(*) one substep of each (2048^2 developed; 128^2 at 0.3 s, third chained substep) has a node whose velocity differs from
the fp64 oracle's by that fraction of the largest node velocity, identically in the engine and the fp32 oracle.  That
node's fp64 mass is 4.9e-14 (2048^2) and 2.2e-9 (128^2) of the heaviest node's: its mass comes only from weights near 0,
which both evaluate with the reference's expanded quadratic 0.5 t^2 - 1.5 t + 1.125, about 1e-7 absolute in fp32, so its
weighted mean velocity is not resolved in fp32.  grid_vel there is held by the yardstick alone; grid_vel_heavy (nodes of
at least 1e-4 of the heaviest node's mass) stays inside the common bound on both substeps and keeps the node velocities
checked.  At rest the fp32 oracle's velocity errors are 1e-3 to 4e-3 and the engine's stay under the common bounds.

test_large_grids also checks the ordering's live count: each substep adds exactly the live rows to the update counter
(bench_2d's rate is made of it) and num_particles is the survivors.  With key_bits one short the dead key res0 res1 = 2^k
aliases cell 0, dead rows sort first and count as live while every position stays right; only those two checks see it.
"""
import time

import numpy as np
import pytest

import bench_2d
from oracle import pyoracle2d as O
from taichi_mpm_b200 import scenes
from tests import common as T
from tests import mpm2d_common as MC
from tests import test_gpu_mpm2d as M

pytestmark = pytest.mark.gpu


def bench_substeps(dt):
    """(at rest, developed) substep counts of bench_2d.py's two measurements, from its argparse defaults (--warmup 20,
    --steps 200, --stage-steps 20, --develop-time 0.05): at rest is the end of the warm-up; developed is the end of the
    developed timed region, after the resting window and its profiled steps (warmup + steps + stage_steps), the develop
    substeps and the timed steps."""
    warmup, steps, stage_steps, develop_time = 20, 200, 20, 0.05
    return warmup, warmup + steps + stage_steps + int(round(develop_time / dt)) + steps


def _checked_substep(e, scene, S_seed, S, label, guards=None):
    """One substep of e from its downloaded state S against the fp64 oracle (compare2d with the yardstick rule); with guards,
    MC.regime2d of S from the same oracle substep must exceed them."""
    oracle = O.substep2d(scene, MC.state_of(S), np.float64)
    if guards is not None:
        r = MC.regime2d(S_seed, S, oracle[0], oracle[1], scene)
        print(label, "regime", r)
        bad = {k: (r[k], g) for k, g in guards.items() if not r[k] > g}
        assert not bad, (label, "regime", bad)
    err, _, _ = M.compare2d(e, scene, MC.state_of(S), ids=S["id"], yardstick=True, oracle=oracle)
    M.assert_parity_yardstick(err, label=label)


# ---------------------------------------------------------------------------------------------------- full size
@pytest.mark.needs_cuda
@pytest.mark.parametrize("state", ["rest", "developed"])
@pytest.mark.parametrize("res", [1024, 2048])
def test_bench_state_full_size(res, state):
    st, dt, scene = MC.bench_column(res)
    rest, developed = bench_substeps(dt)
    n = rest if state == "rest" else developed
    t0 = time.time()
    e = bench_2d.engine_for(res, st, dt, 0)
    e.substep(n)
    _checked_substep(e, scene, st, e.download(), "bench_2d %d^2 %s (substep %d, %.0f s)" % (res, state, n, time.time() - t0),
                     MC.GUARDS_FULL[res] if state == "developed" else None)
    e.close()


@pytest.mark.needs_cuda
@pytest.mark.parametrize("res", [1024, 2048])
def test_full_size_invariants(res):
    st, dt, scene = MC.bench_column(res)
    _, developed = bench_substeps(dt)
    n = len(st["x"])
    a = bench_2d.engine_for(res, st, dt, 0)
    a.substep(developed)
    A = a.download()
    a.close()
    # the same upload, its first substep stage by stage: the P2G grid holds the particle mass and the momentum M g dt (the
    # column is at rest, F = I and apic_b = 0: every particle carries m g dt, and the quadratic weights' first moments vanish)
    b = bench_2d.engine_for(res, st, dt, 0)
    b.sort_particles_and_populate_grid()
    b.rasterize()
    g = b.download_grid(0).astype(np.float64)
    mass = st["mass"].astype(np.float64).sum()
    p = g[..., :2].sum((0, 1))
    want = mass * np.array(scene["gravity"]) * dt
    print("first P2G: mass %.9g of %.9g, momentum %s of %s" % (g[..., 3].sum(), mass, p, want))
    assert abs(g[..., 3].sum() - mass) <= T.TOL_GRID_REL * mass
    assert np.abs(p - want).max() <= T.TOL_GRID_REL * np.abs(want).max()
    b.resample()
    b.substep(developed - 1)
    B = b.download()
    b.close()
    for k in A:
        assert np.array_equal(A[k], B[k]), ("two engines from one upload differ", k)
    ids = A["id"].astype(np.int64)
    assert len(ids) == n and np.array_equal(ids, np.arange(n))   # nothing is deleted in 0.05 s at full size
    assert np.array_equal(A["mass"], st["mass"][ids]) and np.array_equal(A["vol"], st["vol"][ids])
    for k in ("x", "v", "F", "b", "ps"):
        assert np.isfinite(A[k]).all(), k
    # host launches against graph replay, 20 substeps from the developed state
    outs = []
    for no_graph in (False, True):
        e = M.make_engine2d(scene, MC.state_of(A), no_graph=no_graph)
        e.substep(20)
        outs.append(e.download())
        e.close()
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), ("no_graph differs from graph replay", k)


# ---------------------------------------------------------------------------------------------------- reduced size
REDUCED = [pytest.param(res, t, id="%d-%gs" % (res, t), marks=() if res == 64 else pytest.mark.needs_cuda) for res, t in MC.GUARDS_REDUCED]


@pytest.mark.parametrize("res,t", REDUCED)
def test_reduced_developed_collapse(res, t):
    st, dt, scene = MC.bench_column(res)
    n = int(round(t / dt))
    t0 = time.time()
    e = bench_2d.engine_for(res, st, dt, 0)
    e.substep(n)
    S = e.download()
    if t >= 0.3:   # the flow has reached the side bands: particles were deleted there
        assert len(S["id"]) < len(st["x"]), len(S["id"])
    for k in range(3):
        _checked_substep(e, scene, st, S if k == 0 else e.download(), "collapse %d^2 at %g s + %d (%.0f s)" % (res, t, k, time.time() - t0),
                         MC.GUARDS_REDUCED[(res, t)] if k == 0 else None)
    e.close()


# ---------------------------------------------------------------------------------------------------- large grids
# (res, dx): 2^20 cells with a 1-node last tile; 2^22 cells (square and not); dx not a power of two, where X = x / dx
# rounds in fp32, on nnode 2048 (full tiles) x 2051 (a 3-node last tile) and on 1001 x 1537
LARGE = {"1024x1024": ((1024, 1024), 2.0 ** -10), "2048x2048": ((2048, 2048), 2.0 ** -11), "4096x1024": ((4096, 1024), 2.0 ** -12),
         "2047x2050": ((2047, 2050), 0.9 / 2047), "1000x1536": ((1000, 1536), 1.0 / 1000)}
LARGE_CASES = [(name, 1) for name in LARGE] + [("2048x2048", 0), ("4096x1024", 0)]


def large_scene(res, dx, clean):
    """Sand blocks of 8 x 8 cells in the four corners, one cell from the faces (they start in the 7-cell band), moving outwards
    at up to 0.8 cells per substep, so that with clean_boundary = 0 the upper faces' stencil rule deletes too, and one block
    across a tile edge in the middle; gravity with two components.  The upper corners reach the last node tile on both
    axes."""
    r0, r1 = res
    blocks = [((x0, y0), (x0 + 8, y0 + 8)) for x0 in (1, r0 - 9) for y0 in (1, r1 - 9)]
    mid = (16 * (r0 // 32) - 4, 16 * (r1 // 32) - 4)
    blocks.append((mid, (mid[0] + 8, mid[1] + 8)))
    scene, st = MC.scene2d(scenes.MAT_SAND, res=res, dx=dx, blocks=blocks, gravity=(3.0, -8.0), levelset=None, clean_boundary=clean, seed=40)
    X = st["x"].astype(np.float64) / scene["dx"]
    out = (X - np.array(res) / 2.0) / (np.array(res) / 2.0)
    st["v"] = (st["v"] + out * 0.8 * scene["dx"] / scene["dt"]).astype(np.float32)
    return scene, st


@pytest.mark.parametrize("name,clean", LARGE_CASES, ids=["%s-clean%d" % c for c in LARGE_CASES])
def test_large_grids(name, clean):
    res, dx = LARGE[name]
    scene, st = large_scene(res, dx, clean)
    e = M.make_engine2d(scene, st)
    deleted = []
    for k in range(3):
        now = e.download()
        u0 = e.update_count()
        err, got, _ = M.compare2d(e, scene, st if k == 0 else MC.state_of(now), ids=None if k == 0 else now["id"], check_grid=(k == 0),
                                    yardstick=True)
        M.assert_parity_yardstick(err, grid=(k == 0), label="%s clean_boundary %d, substep %d" % (name, clean, k))
        # the ordering found exactly the live rows: the dead rows (key res0 res1) sorted after them.  Dead rows sorted
        # anywhere else still leave every position right, but count as live in the updates bench_2d's rate is made of.
        assert e.update_count() - u0 == len(now["id"]), (k, e.update_count() - u0, len(now["id"]))
        assert e.num_particles() == len(got["id"])
        deleted.append(len(now["id"]) - len(got["id"]))
    e.close()
    assert deleted[0] > 0, deleted   # dead rows keep their storage: the second and third orderings sort them
