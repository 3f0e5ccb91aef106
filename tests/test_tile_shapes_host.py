"""The guards of tests/tile_shapes.py on the fp64 oracle's trajectory of the tile-walk scene: the scene reaches every
required edge category, and a scene that lost one (run lengths rounded to multiples of 64) is caught."""
import numpy as np

from oracle import pyoracle as O
from tests import tile_shapes as TS


def _oracle_states(scene, st):
    """The states before and after each of NSUB oracle substeps, as the engine would download them (ids, alive only)."""
    ids = np.arange(len(st["x"]))
    cur = dict(st)
    states = [dict(id=ids, x=st["x"])]
    for _ in range(TS.NSUB):
        ref, _, _ = O.substep(scene, cur, np.float64, want_grids=False)
        alive = ref["alive"].astype(bool)
        cur = {k: np.asarray(ref[k])[alive].astype(np.float32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        cur["group"] = ref["group"][alive]
        ids = ids[alive]
        states.append(dict(id=ids, x=cur["x"]))
    return states


def test_the_tile_walk_scene_reaches_every_edge_category():
    miss, min_active = TS.missing(_oracle_states(*TS.tile_scene()))
    assert not miss, miss
    assert min_active >= 8 * TS.G2P_CTAS_PER_SM * 3, min_active


def test_the_guards_catch_a_scene_without_the_run_length_edges():
    rounded = tuple(max(64, 64 * int(round(n / 64))) for n in TS.RUN_LENGTHS)
    miss, _ = TS.missing(_oracle_states(*TS.tile_scene(run_lengths=rounded)))
    assert {("run_len", n) for n in (127, 129, 511, 513, 1151, 1153)} <= set(miss), miss
