"""The window rule of tests/collapse.py on a sand column the fp32 port has settled onto its floor (no GPU): the fp64
oracle's substep of a window of the state equals its substep of the whole state on the compared particles and nodes, and a
margin of one node is not enough.  The GPU legs (tests/test_gpu_zz_collapse_parity.py) check an 8 M state through such
windows."""
import functools

import numpy as np
import pytest

from oracle import pyoracle as O
from tests import collapse as CL

SCALE = 0.125        # 32^3, 13 824 particles
# port substeps (16-30 s on 8 cores).  0.04 s of flow: the column has compressed onto the floor (its centre of mass is
# 0.13 cells lower, its floor nodes stick and slide, its sand is in return-map cases 0 and 2) but has not spread
# (footprint 1.0x, no particle in case 1, at most 12 per cell).  It is a settled column, not the developed collapse.
DEVELOP = 2000


@functools.lru_cache(maxsize=1)
def developed():
    scene, S = CL.port_collapse(SCALE, DEVELOP)
    S = {k: v for k, v in S.items() if k != "id"}
    return scene, S, O.substep(scene, S, np.float64)


def windows(S, dx, res):
    """Node boxes of 8^3 by rule: on the floor at the pile's edge, at the free surface above its centre, at its densest cell."""
    base = CL.base_nodes(S["x"], dx)
    low = base[:, 1] <= base[:, 1].min() + 1
    c = base.mean(0)
    toe = base[low][np.argmax(np.abs(base[low][:, 0] - c[0]))]
    top = base[np.argmax(base[:, 1] - 2 * np.abs(base[:, [0, 2]] - c[[0, 2]]).sum(1))]
    cells, counts = np.unique(base, axis=0, return_counts=True)
    dense = cells[np.argmax(counts)]
    return dict(toe=CL.clip_box(toe, 8, res), surface=CL.clip_box(top, 8, res), densest=CL.clip_box(dense, 8, res))


def _errors(S, ref_all, g_all, gv_all, lo, hi, margin, dx):
    sub, mask, nodes = CL.window(S, lo, hi, margin, dx=dx)
    ref, g, gv = O.substep(dict(developed()[0]), sub, np.float64)
    whole = np.nonzero(((CL.base_nodes(S["x"], dx) >= lo) & (CL.base_nodes(S["x"], dx) < hi)).all(1))[0]
    err = {}
    for k in ("x", "v", "F", "b", "ps"):
        a, b = ref[k][mask], ref_all[k][whole]
        err[k] = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))
    for name, a, b in (("grid", g, g_all), ("grid_vel", gv, gv_all)):
        a, b = CL.box(a, nodes), CL.box(b, nodes)
        err[name] = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))
    assert np.array_equal(ref["alive"][mask], ref_all["alive"][whole])
    return err, int(mask.sum())


def test_port_state_is_a_settled_column():
    # about half of each measured value: com_drop 0.127 cells, 32 sticking and 238 sliding floor nodes, 1 184 / 12 640
    # particles in return-map cases 0 / 2, largest logJp 1.0e-3
    scene, S, (ref, g, _) = developed()
    _, _, S0 = CL.seeded_state(SCALE)
    r = CL.regime(S0, S, S, ref, g, scene, dict(movers=0, rows=1))
    print("port-settled 32^3 column", r)
    assert r["stick"] > 16 and r["slide"] > 119, r
    assert r["case0"] > 590 and r["case2"] > 6300 and r["ps_max"] > 5e-4, r
    assert r["com_drop"] > 0.06, r


@pytest.mark.parametrize("where", ["toe", "surface", "densest"])
def test_window_substep_equals_whole_substep(where):
    scene, S, (ref_all, g_all, gv_all) = developed()
    lo, hi = windows(S, scene["dx"], scene["res"])[where]
    err, n = _errors(S, ref_all, g_all, gv_all, lo, hi, CL.MARGIN, scene["dx"])
    print(where, lo, n, err)
    assert n > 200
    assert max(err.values()) <= 1e-12, err
    # one node of margin drops particles that scatter into the window's first node layer: the check sees them missing
    err1, _ = _errors(S, ref_all, g_all, gv_all, lo, hi, 1, scene["dx"])
    print(where, "margin 1", err1)
    assert err1["v"] > 1e-5 and err1["b"] > 1e-3 and err1["grid"] > 1e-3, err1
