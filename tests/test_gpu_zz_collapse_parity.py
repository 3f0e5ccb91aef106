"""The developed sand collapse that bench.py times, against the fp64 oracle, substep by substep.

bench.py's `value` is the slower of sand256 at rest (after 20 substeps) and after the collapse has developed (its timed
region ends at substep 20 640, tests/collapse.py).  There the pile is compacted at its bottom, its floor nodes take both
Coulomb branches, its sand sits in every case of the return map, most of it is nearly at rest, and the cached affine matrix
and the incremental ordering are what 20 000 graph-replayed substeps left behind.  These tests reach that state on the
engine's own path (mpmb_seed_lattice, then e.substep(n), never an upload) and check it:

- test_reduced_collapse_chained: 64^3 and 128^3, at substeps 20, 2 000 and 20 640: three chained substeps against the
  oracle's substep of the engine's own state (test_gpu_tile_walk.chain) and the next P2G against the stress part
  (test_gpu_next_p2g.next_p2g); the regime guards at 20 640.
- test_full_size_bench_state: 256^3, 8 M particles, at substeps 20 and 20 640: one substep against the fp32 port on every
  particle, and the same substep stage by stage against the fp64 oracle on windows chosen by rule (the toe of the pile,
  its densest cell, its free surface, its fastest particle), the next P2G too; the regime guards.
- test_collapse_on_z_slabs: 64^3 cut into 2 and 4 z slabs over the peer-memory path, developed 20 640 substeps; one
  substep of the union against the oracle.
- test_port_settled_column_after_upload: a 32^3 column the port settled onto its floor in 2 000 substeps (compressed, not
  spread: tests/test_collapse_window_host.py), uploaded, 4 substeps, then the chained and the window checks; it also runs
  on the SIMT emulator (tests/test_collapse_parity_simt.py), which cannot run the 20 000 substeps of the others.
A window is a node box [lo, hi): the oracle steps the particles whose base node lies within two nodes of it and is then
exact on the particles based inside it and on the nodes [lo, hi + 2) (tests/test_collapse_window_host.py shows both)."""
import os
import time

import numpy as np
import pytest

from oracle import pyoracle as O
from tests import collapse as CL
from tests import common as T
from tests import test_gpu_next_p2g as NP
from tests import test_gpu_tile_walk as TW

pytestmark = pytest.mark.gpu
SIMT = os.environ.get("MPMB_SIMT", "") == "1"

# Tolerances: 4-5x the worst error measured on an H100 80GB HBM3 (700 W) and on the SIMT emulator (DESIGN §2).
# chained substeps: test_gpu_tile_walk's names and normalisations; next = the next P2G against the stress part
TOL_CHAIN = dict(TW.TOL_PROD, grid_vel=1.4e-5, v=3e-6, b=7e-5, F=2.4e-6, ps=2.4e-6, stress=4.5e-4, next=4.5e-4)
# the column at rest (substep 20): every particle has fallen for 20 substeps (|v| <= 4e-3 m/s) and the stress part is
# 6e-5 of the grid, so the same absolute fp32 rounding of the P2G sums (grid_rast 3e-7, as in the developed states) is a
# larger fraction of the small velocities and of the stress part that normalise these errors
TOL_REST = dict(TOL_CHAIN, grid_vel=1.5e-3, v=2e-4, b=8e-4, stress=2.5e-3, next=2.5e-3)
# windows: grid = P2G (p, m) relative to the window's largest, grid_vel = heavy-node velocities relative to the window's
# largest, stress = P2G momentum relative to the window's stress part (windows where it is visible), next = the next P2G
# likewise; x absolute, v and b relative to the largest over all particles, F absolute, ps as T.ps_err.  At the toe the
# stress part is only 4e-4 of the window's grid, and the grid's fp32 rounding (5e-7 of it) is 1.3e-3 of the stress part.
TOL_WIN = dict(grid=2.5e-6, grid_vel=4e-5, stress=6e-3, next=6e-3, x=1.5e-7, v=4.5e-6, b=1.2e-4, F=2e-6, ps=2.3e-6)
TOL_WIN_REST = dict(TOL_WIN, grid_vel=3e-3, v=5e-4, b=3e-3, stress=2.5e-3, next=2e-3)
# the fp32 port on all 8 M particles: tests/common.py's single-substep bounds (at rest: relative to |v| <= 4e-3 m/s)
TOL_PORT = dict(x=T.TOL_X_ABS, v=T.TOL_V_REL, b=T.TOL_V_REL, F=T.TOL_F_ABS, ps=T.TOL_PS_ABS)
TOL_PORT_REST = dict(TOL_PORT, v=1e-3, b=5e-3)
# the developed state (substep 20 640): about half of what the first H100 run measured (DESIGN §2)
GUARDS = {0.25: dict(movers=3, stick=500, slide=1400, case0=36000, case1=1100, case2=20000, ppc_max=11, com_drop=4.4,
                     footprint=2.0, resting=0.4, ps_max=0.068),
          0.5: dict(movers=120, stick=2800, slide=6700, case0=250000, case1=28000, case2=198000, ppc_max=15, com_drop=9.0,
                    footprint=2.5, resting=0.4, ps_max=0.056),
          1.0: dict(movers=1900, stick=17000, slide=26000, case0=167000, case1=44000, case2=117000, ppc_max=23, com_drop=18.0,
                    footprint=2.8, resting=0.4, ps_max=0.11)}
WIN = 24           # window size in nodes at full size
SELECT = ("toe", "densest", "surface", "front")


def _fmt(d):
    return {k: ("%.3g" % v if isinstance(v, float) else v) for k, v in d.items()}


def _assert_within(worst, tol, label):
    print(label, _fmt(worst))
    bad = {k: (v, tol[k]) for k, v in worst.items() if k in tol and not v <= tol[k]}
    assert not bad, (label, bad)


def _assert_guards(r, scale):
    bad = {k: (r[k], g) for k, g in GUARDS[scale].items() if not r[k] > g}
    assert not bad, ("regime", scale, bad)


def _merge(worst, err):
    for k, v in err.items():
        worst[k] = max(worst.get(k, 0.0), float(v))


# ---------------------------------------------------------------------------------------------------- windows by rule
def select_windows(S, scene, size):
    """Node boxes around: the pile's toe (the floor particle farthest from the column's axis), its densest cell, its free
    surface above the axis, and its fastest particle (the flowing front)."""
    dx, res = scene["dx"], np.asarray(scene["res"])
    base = CL.base_nodes(S["x"], dx)
    axis = res / 2.0
    horiz = np.sqrt(((base[:, [0, 2]] - axis[[0, 2]]) ** 2).sum(1))
    low = base[:, 1] <= base[:, 1].min() + 1
    toe = base[low][np.argmax(horiz[low])]
    key = (base[:, 0] * (res[1] + 1) + base[:, 1]) * (res[2] + 1) + base[:, 2]
    dense = base[np.argmax(np.bincount(key)[key])]
    top = base[np.argmax(base[:, 1] - 2.0 * horiz)]
    front = base[np.argmax((S["v"].astype(np.float64) ** 2).sum(1))]
    return {k: CL.clip_box(c, size, res) for k, c in zip(SELECT, (toe, dense, top, front))}


def _rows(ids, want):
    """Rows of the id-sorted `ids` that hold `want` (all present)."""
    r = np.searchsorted(ids, want)
    assert (r < len(ids)).all() and np.array_equal(ids[r], want)
    return r


def window_substep(e, scene, boxes, port=False):
    """One substep of e stage by stage, checked on every window of `boxes` against the fp64 oracle: the P2G grid, its stress
    part (the cached affine matrix), the heavy nodes' velocities after k_grid (floor projection included), the particles,
    and the next P2G's stress part.  port=True: also every particle against the fp32 port.  Returns (worst errors, the
    checked state, the oracle's windows of it, counts)."""
    dx = scene["dx"]
    S = e.download()
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g0 = e.download_grid(0)
    g1 = e.download_grid(1)
    e.resample()
    got = e.download()
    worst, counts, near_edge = {}, {}, 0
    for name, (lo, hi) in boxes.items():
        sub, mask, nodes = CL.window(S, lo, hi, dx=dx)
        ref, gr, gv = O.substep(scene, sub, np.float64)
        _, gf, _ = O.substep(scene, NP._free_state(scene, sub), np.float64)
        gr, gv, gf = CL.box(gr, nodes), CL.box(gv, nodes), CL.box(gf, nodes)
        e0, e1 = CL.box(g0, nodes).astype(np.float64), CL.box(g1, nodes).astype(np.float64)
        gmax = max(np.abs(gr[..., :3]).max(), gr[..., 3].max())
        heavy = gr[..., 3] >= 1e-4 * gr[..., 3].max()
        se = NP._grid_errors(e0, gr, gf)
        err = dict(grid=np.abs(e0 - gr).max() / gmax, visible=se["visible"],
                   grid_vel=(np.abs(e1[..., :3] - gv[..., :3]).max(-1)[heavy]).max() / np.abs(gv[..., :3]).max())
        assert not e0[gr[..., 3] == 0].any(), (name, "mass outside the oracle's active nodes")
        # particles based in the window: the alive sets agree, except within fp32 rounding of the clean_boundary band
        ids = sub["id"][mask]
        alive = ref["alive"][mask].astype(bool)
        have = np.isin(ids, got["id"])
        if not np.array_equal(have, alive):
            X = ref["x"][mask][have != alive] / dx
            edge = np.minimum(np.abs(X - 7.0), np.abs(X - (np.asarray(scene["res"]) - 7.0))).min(1)
            assert (edge < 1e-5).all(), (name, "alive sets differ away from the band edge", ids[have != alive])
            near_edge += int((have != alive).sum())
        keep = alive & have
        g = {k: got[k][_rows(got["id"], ids[keep])] for k in ("x", "v", "F", "b", "ps")}
        r = {k: ref[k][mask][keep] for k in ("x", "v", "F", "b", "ps")}
        err.update(x=np.abs(g["x"] - r["x"]).max(), v=np.abs(g["v"] - r["v"]).max() / np.abs(got["v"]).max(),
                   b=np.abs(g["b"] - r["b"]).max() / np.abs(got["b"]).max(), F=np.abs(g["F"] - r["F"]).max(), ps=T.ps_err(g["ps"], r["ps"]))
        counts[name] = dict(lo=[int(v) for v in lo], particles=int(mask.sum()), nodes=int((gr[..., 3] > 0).sum()))
        if se["visible"] >= TW.VISIBLE:   # at rest the stress has not reached the top of the column yet
            err["stress"] = se["stress"]
            counts["stress_windows"] = counts.get("stress_windows", 0) + 1
        print("  window %s" % name, counts[name], _fmt({k: float(v) for k, v in err.items()}))
        err.pop("visible")
        _merge(worst, err)
    counts["alive_differ_at_band_edge"] = near_edge
    if port:   # every particle against the fp32 port of the reference's optimized path
        f = O.FastOracle(scene, S)
        f.substeps(1)
        alive = f.st["alive"].astype(bool)
        assert np.array_equal(got["id"], S["id"][alive]), "the port deletes other particles"
        pr = {k: f.st[k][alive] for k in ("x", "v", "F", "b", "ps")}
        pe = dict(x=np.abs(got["x"] - pr["x"]).max(), v=np.abs(got["v"] - pr["v"]).max() / np.abs(pr["v"]).max(),
                  b=np.abs(got["b"] - pr["b"]).max() / np.abs(pr["b"]).max(), F=np.abs(got["F"] - pr["F"]).max(),
                  ps=np.abs(got["ps"] - pr["ps"]).max())
        worst.update({"port_" + k: float(v) for k, v in pe.items()})
        del f
    # the next P2G: the cached affine matrix k_g2p wrote in this substep
    S2 = e.download()
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g0 = e.download_grid(0)
    e.resample()
    for name, (lo, hi) in boxes.items():
        sub, _, nodes = CL.window(S2, lo, hi, dx=dx)
        _, gr, _ = O.substep(scene, sub, np.float64)
        _, gf, _ = O.substep(scene, NP._free_state(scene, sub), np.float64)
        se = NP._grid_errors(CL.box(g0, nodes).astype(np.float64), CL.box(gr, nodes), CL.box(gf, nodes))
        if se["visible"] >= TW.VISIBLE:
            _merge(worst, dict(next=se["stress"]))
    return worst, S, counts


def floor_regime(e, scene, S_seed, S, stats):
    """collapse.regime with the oracle's P2G grid of the floor band (a window over the whole x-z extent)."""
    lo, hi = CL.floor_box(scene)
    sub, _, _ = CL.window(S, lo, hi, dx=scene["dx"])
    ref, gr, _ = O.substep(scene, sub, np.float64)
    return CL.regime(S_seed, S, sub, ref, gr, scene, stats)


# ---------------------------------------------------------------------------------------------------- a: reduced, chained
@pytest.mark.parametrize("scale", [0.25, 0.5], ids=["64", "128"])
def test_reduced_collapse_chained(scale):
    if SIMT:
        pytest.skip("20 000 substeps: the emulator runs the port-settled column instead")
    e, scene, meta, n = CL.seeded_engine(scale)
    _, _, S_seed = CL.seeded_state(scale)
    assert n == len(S_seed["x"])
    done, report = 0, {}
    for cp in (CL.QUIESCENT, 2000, CL.DEVELOPED):
        t0 = time.time()
        e.substep(cp - done)
        stats = e.get_ordering_stats()
        S = e.download()
        ref, gr, _ = O.substep(scene, S, np.float64)
        r = CL.regime(S_seed, S, S, ref, gr, scene, stats)
        worst, _ = TW.chain(e, scene, 3, stress=True, all_nodes=False)
        err, _ = NP.next_p2g(e, scene, "collapse %d^3 at %d: next P2G" % (scene["res"][0], cp), tol=1.0, guard=TW.VISIBLE)
        worst["next"] = err["stress"]
        done = cp + 4
        print("collapse %d^3 at substep %d (%.0f s)" % (scene["res"][0], cp, time.time() - t0), "regime", _fmt(r))
        report[cp] = (worst, r)
    e.close()
    for cp, (worst, r) in report.items():
        print("collapse %d^3 at %d" % (scene["res"][0], cp), _fmt(worst))
    for cp, (worst, r) in report.items():
        _assert_within(worst, TOL_REST if cp == CL.QUIESCENT else TOL_CHAIN, "collapse %d^3 at %d" % (scene["res"][0], cp))
    _assert_guards(report[CL.DEVELOPED][1], scale)


# ---------------------------------------------------------------------------------------------------- b: full size
@pytest.mark.needs_cuda
def test_full_size_bench_state():
    if SIMT:
        pytest.skip("8 M particles")
    e, scene, meta, n = CL.seeded_engine(1.0)
    _, _, S_seed = CL.seeded_state(1.0)
    assert n == len(S_seed["x"]) == 8_000_000
    done, report = 0, {}
    for cp in (CL.QUIESCENT, CL.DEVELOPED):
        t0 = time.time()
        e.substep(cp - done)
        stats = e.get_ordering_stats()
        S = e.download()
        boxes = select_windows(S, scene, WIN)
        r = floor_regime(e, scene, S_seed, S, stats)
        print("sand256 at substep %d, regime" % cp, _fmt(r))
        worst, _, counts = window_substep(e, scene, boxes, port=True)
        done = cp + 2
        print("sand256 at substep %d (%.0f s)" % (cp, time.time() - t0), _fmt(worst), counts)
        report[cp] = (worst, r, counts)
    e.close()
    for cp, (worst, r, counts) in report.items():
        print("sand256 at %d" % cp, _fmt(worst), _fmt(r))
    for cp, (worst, r, counts) in report.items():
        tol = TOL_WIN_REST if cp == CL.QUIESCENT else TOL_WIN
        _assert_within({k: v for k, v in worst.items() if not k.startswith("port_")}, tol, "sand256 windows at %d" % cp)
        assert counts.get("stress_windows", 0) >= (2 if cp == CL.QUIESCENT else 4), counts
        _assert_within({k[5:]: v for k, v in worst.items() if k.startswith("port_")}, TOL_PORT_REST if cp == CL.QUIESCENT else TOL_PORT,
                       "sand256 vs port at %d" % cp)
        assert counts["alive_differ_at_band_edge"] == 0, counts
        for name in SELECT:
            assert counts[name]["particles"] > 1000, counts
    _assert_guards(report[CL.DEVELOPED][1], 1.0)


# ---------------------------------------------------------------------------------------------------- c: z slabs
@pytest.mark.parametrize("world", [2, 4])
def test_collapse_on_z_slabs(world):
    if SIMT:
        pytest.skip("20 000 substeps")
    S = CL.SeededSlabs(0.25, world)
    t0 = time.time()
    S.step(CL.DEVELOPED)
    U = S.union()
    ref, _, _ = O.substep(S.scene, U, np.float64, want_grids=False)
    NP._slab_next_p2g(S, S.scene, "collapse on %d slabs" % world)
    got = S.union()
    S.close()
    alive = ref["alive"].astype(bool)
    assert np.array_equal(got["id"], U["id"][alive])
    r = {k: ref[k][alive] for k in ("x", "v", "F", "b", "ps")}
    err = dict(x=np.abs(got["x"] - r["x"]).max(), v=np.abs(got["v"] - r["v"]).max() / np.abs(r["v"]).max(),
               b=np.abs(got["b"] - r["b"]).max() / np.abs(r["b"]).max(), F=np.abs(got["F"] - r["F"]).max(), ps=T.ps_err(got["ps"], r["ps"]))
    print("collapse on %d slabs, cuts %s, %d of %d particles (%.0f s)" % (world, S.cuts, len(U["id"]), S.n, time.time() - t0))
    _assert_within(err, TOL_CHAIN, "collapse on %d slabs vs oracle" % world)


# ---------------------------------------------------------------------------------------------------- d: port-settled, uploaded
PORT_SCALE, PORT_DEVELOP = 0.125, 2000


def test_port_settled_column_after_upload():
    from tests.test_collapse_window_host import developed, windows
    scene, S, _ = developed()
    t0 = time.time()
    e = T.make_engine(scene, S)
    movers = 0
    for _ in range(4):   # movers, holes and arrivals of the incremental ordering exist again
        e.substep(1)
        movers += e.get_ordering_stats()["movers"]
    worst, _ = TW.chain(e, scene, 3, stress=True, all_nodes=False)
    boxes = windows(e.download(), scene["dx"], scene["res"])
    w, _, counts = window_substep(e, scene, boxes)
    e.close()
    print("port-settled 32^3 after upload (%.0f s, %d movers)" % (time.time() - t0, movers), counts)
    _assert_within(worst, TOL_CHAIN, "port-settled 32^3, chained")
    _assert_within(w, TOL_WIN, "port-settled 32^3, windows")
    assert movers > 0 and counts.get("stress_windows", 0) == 3, (movers, counts)
