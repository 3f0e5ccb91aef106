"""k_p2g, k_grid and k_g2p when every CTA (every k_grid warp) walks many tiles, against the fp64 oracle.

The persistent grids are sized from the device (k_p2g SMs x 4, k_g2p SMs x 5, k_grid SMs x 8 CTAs of 8 warps), so on an
H100 a scene of a few hundred tiles gives each CTA at most the tile at its block index: the claim loops, k_g2p's
one-tile-ahead claim, the s_vel / s_stay double buffers, the mbarrier parity carried across tiles and k_grid's
`slot += nw` loop never run.  MPMB_NUM_SMS=k sizes every launch for min(k, SMs) SMs instead; with k = 1 the scene of
tests/tile_shapes.py (about 300 active tiles) gives each of k_g2p's five CTAs about 60 tiles.  That scene places tiles at
the chunk edges of both kernels, at every run / arrival split and every outpos alignment shift, and its guards fail if a
category stops occurring.

- test_chained_substeps_match_the_oracle: six substeps, each against the oracle's substep of the engine's own state.
- test_grid_size_changes_no_bit: every path without float atomics gives the same bits for k = 1, 3, 7 and unset.
- test_existing_oracle_files_pass_with_one_sm: the oracle-checked files again, with MPMB_NUM_SMS=1.
- test_production_grid_walks_several_tiles: a 128^3 scene with more tiles than k_grid has warps, without the hook.
- test_bounds_checked_build_reports_nothing: the chained test and the slab leg on the -DMPMB_CHECKED build, one SM.
Runs on the SIMT emulator too (tests/test_tile_walk_simt.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pyoracle as O
from taichi_mpm_b200 import capi, scenes
from tests import common as T
from tests import tile_shapes as TS
from tests.test_gpu_next_p2g import _free_state, _grid_errors

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT = os.environ.get("MPMB_SIMT", "") == "1"
KEYS = ("id", "x", "v", "F", "b", "ps")

# Tolerances of the chained comparison (worst errors measured on an H100 and on the emulator: DESIGN §2)
TOL = dict(grid_rast=1e-6, grid_vel=7e-6, grid_vel_all=1e-2, x=1.5e-7, v=1.5e-6, b=5e-5, F=4e-6, ps=1.5e-6, stress=1.5e-4)
# the production scene's node and particle velocities (measured worst 7.7e-6 and 2.5e-6 on the H100)
TOL_PROD = dict(TOL, grid_vel=3.5e-5, v=1.2e-5)
VISIBLE = 3e-5      # the stress part must be at least this fraction of the grid's largest momentum or mass


def _hook(monkeypatch, k):
    if k is None:
        monkeypatch.delenv("MPMB_NUM_SMS", raising=False)
    else:
        monkeypatch.setenv("MPMB_NUM_SMS", str(k))


def chain(e, scene, nsub, stress=True, all_nodes=True):
    """nsub substeps of engine e stage by stage, each checked against the oracle's substep of e's downloaded state.
    Returns (worst error of each quantity, the states before and after every substep, for the layout guards)."""
    worst = {}
    states = []
    for s in range(nsub):
        S = e.download()
        states.append(S)
        ref, g_rast, g_vel = O.substep(scene, S, np.float64)
        e.sort_particles_and_populate_grid()
        e.rasterize()
        g0 = e.download_grid(0).astype(np.float64)
        g1 = e.download_grid(1).astype(np.float64)
        e.resample()
        got = e.download()
        alive = ref["alive"].astype(bool)
        assert np.array_equal(got["id"], S["id"][alive]), "substep %d: alive set" % (s + 1)
        gmax = max(np.abs(g_rast[..., :3]).max(), g_rast[..., 3].max())
        active = g_rast[..., 3] > 0
        # node velocities: tightly where the mass is at least 1e-4 of the largest, loosely at every active node.  At a
        # stencil corner of a lone particle the mass is ~1e-9 of the largest, and momentum / mass there turns fp32 rounding
        # of the weights into errors of ~1e-3 (no particle sees that node with more than that weight).  all_nodes=False:
        # the tight check only (at the lightest nodes of the production scene's sparse tiles the fp32 node velocity is off
        # by 0.67 of the largest velocity on an H100: no significant digit is left there)
        heavy = g_rast[..., 3] >= 1e-4 * g_rast[..., 3].max()
        dv = np.abs(g1[..., :3] - g_vel[..., :3]) / np.abs(g_vel[..., :3]).max()
        err = dict(grid_rast=np.abs(g0 - g_rast).max() / gmax, grid_vel=dv[heavy].max())
        if all_nodes:
            err["grid_vel_all"] = dv[active].max()
        assert not g0[~active].any(), "substep %d: mass outside the oracle's active nodes" % (s + 1)
        r = {k: ref[k][alive] for k in ("x", "v", "b", "F", "ps")}
        err["x"] = np.abs(got["x"] - r["x"]).max()
        err["v"] = np.abs(got["v"] - r["v"]).max() / np.abs(r["v"]).max()
        err["b"] = np.abs(got["b"] - r["b"]).max() / np.abs(r["b"]).max()
        err["F"] = np.abs(got["F"] - r["F"]).max()
        err["ps"] = T.ps_err(got["ps"], r["ps"])
        if stress:   # the P2G grid against the stress part: the affine matrix the previous k_g2p cached
            _, g_free, _ = O.substep(scene, _free_state(scene, S), np.float64)
            se = _grid_errors(g0, g_rast, g_free)
            assert se["visible"] >= VISIBLE, se
            err["stress"] = se["stress"]
        for k, v in err.items():
            worst[k] = max(worst.get(k, 0.0), float(v))
    states.append(e.download())
    return worst, states


def _assert_within(worst, label, tol=TOL):
    print(label, {k: "%.3g" % v for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= tol[k], (label, k, v)


def _assert_guards(states, ctas):
    miss, min_active = TS.missing(states)
    assert not miss, "edge categories not reached: %s" % miss
    assert min_active >= 8 * ctas, (min_active, ctas)


# ---------------------------------------------------------------------------------------------------- a: chained parity
@pytest.mark.parametrize("k", [1, 3, None], ids=["sms1", "sms3", "unset"])
def test_chained_substeps_match_the_oracle(k, monkeypatch):
    _hook(monkeypatch, k)
    scene, st = TS.tile_scene()
    e = T.make_engine(scene, st)
    worst, states = chain(e, scene, TS.NSUB)
    e.close()
    _assert_within(worst, "tile walk, MPMB_NUM_SMS=%s" % k)
    _assert_guards(states, TS.G2P_CTAS_PER_SM * 3)   # at least 8 tiles per k_g2p CTA up to k = 3


# ---------------------------------------------------------------------------------------------------- b: bit for bit
# Which launches sized from num_sms each leg reaches (the rigid kernels add with float atomics: the oracle files of c):
#   sequence   k_mover_place, k_mover_rank, k_p2g, k_grid, k_g2p (with and without apic_b, both parts), graph replay
#   tile scene k_p2g, k_grid, k_g2p at every chunk edge, k_dense_grid (download_grid)
#   slabs      k_halo_pack, k_halo_unpack, k_migrate_pack (2 slabs, host-moved buffers), k_halo_send2, k_halo_recv2,
#              k_migrate_send2 (2 and 4 slabs, peer memory), k_layer_hist, k_recut_check, k_recut_keep (the re-cut)
#   seed       k_seed_flags, k_seed_write, k_shapes_to_sdf, k_planes_to_sdf, k_count_live (delete_inside_levelset)
#   async      the AsyncMPM device advance (sized from its blocks, not from num_sms: it must not notice the hook)
def _leg_sequence():
    from tests.test_tile_claims import run_sequence
    return run_sequence(no_graph=False) + run_sequence(no_graph=True)


def _leg_tile_scene():
    scene, st = TS.tile_scene()
    e = T.make_engine(scene, st)
    e.substep(3)
    out = [{k: e.download()[k] for k in KEYS}]
    e.sort_particles_and_populate_grid()
    e.rasterize()
    out.append({"grid0": e.download_grid(0), "grid1": e.download_grid(1)})
    e.resample()
    e.close()
    return out


def _leg_slabs():
    # 2 slabs through the host-moved buffers (k_halo_pack / unpack, k_migrate_pack), 2 and 4 over peer memory; each
    # drifts, takes an append, is re-cut as slab.rebalance does it and runs on
    from tests.test_gpu_slab import _scene
    from tests.test_gpu_slab_recut import _drifted, _recut
    scene, st = _scene()
    out = []
    for world, peer in ((2, False), (2, True), (4, True)):
        S, ref = _drifted(scene, st, world, peer, steps=4)
        ref.close()
        _recut(S)
        S.step(3)
        out += [{k: p[k] for k in KEYS} for p in S.parts()]
        S.close()
    return out


def _leg_seed():
    e = capi.Engine((32, 32, 32), 1.0 / 32, 2e-5, (0.0, -10.0, 0.0), True, True)
    e.set_material(0, scenes.MAT_SAND, scenes.material_params(scenes.MAT_SAND))
    e.set_levelset_shapes([(capi.SHAPE_PLANE, False, [0.0, 1.0, 0.0, -9.6]), (capi.SHAPE_SPHERE, False, [16.0, 14.0, 16.0, 3.2])], 0.4)
    e.seed_lattice((9, 10, 9), (23, 20, 23), (1.0 / 32) ** 3 / 8, 400.0 * (1.0 / 32) ** 3 / 8, jitter=0.2, seed=3, v0=(0.5, -1.0, 0.2))
    e.delete_inside_levelset()
    e.substep(4)
    out = [{k: e.download()[k] for k in KEYS}]
    e.set_planes(np.array([[0.0, 1.0, 0.0, -11.6]], np.float32), 0.4)
    e.delete_inside_levelset()
    e.substep(2)
    out.append({k: e.download()[k] for k in KEYS})
    e.close()
    return out


def _leg_async():
    from taichi_mpm_b200 import async_mpm
    scene, st = T.perturbed_scene(scenes.MAT_SAND, res=32, cells=8, seed=7, strain=0.0, vel=0.0, with_floor=False)
    unit = 5e-6
    m = async_mpm.AsyncMPM(res=(32, 32, 32), base_delta_t=unit, unit_delta_t=unit, max_units=64, cfl_dt_mul=0.1, gravity=scene["gravity"])
    assert m._device_pools
    m.add_particles(type="sand", positions=st["x"], density=400.0)
    v = np.zeros_like(st["v"])
    v[st["x"][:, 0] > 0.55, 0] = 10.0
    m.pool["v"][:] = v
    for _ in range(2):
        m.step(80 * unit)
    p = m.get_particles()
    return [{k: np.asarray(p[k]) for k in p}]


LEGS = dict(sequence=_leg_sequence, tile_scene=_leg_tile_scene, slabs=_leg_slabs, seed=_leg_seed, async_device=_leg_async)


def _same(a, b, what):
    assert len(a) == len(b), what
    for i, (sa, sb) in enumerate(zip(a, b)):
        assert sorted(sa) == sorted(sb), what
        for k in sa:
            x, y = np.ascontiguousarray(sa[k]), np.ascontiguousarray(sb[k])
            assert x.shape == y.shape and x.tobytes() == y.tobytes(), "%s: part %d, %s" % (what, i, k)


@pytest.mark.parametrize("leg", sorted(LEGS))
def test_grid_size_changes_no_bit(leg, monkeypatch):
    _hook(monkeypatch, None)
    base = LEGS[leg]()
    # the emulator has 2 SMs: 3 and 7 clamp to 2, the same grids as unset
    for k in ((1,) if SIMT else (1, 3, 7)):
        _hook(monkeypatch, k)
        _same(base, LEGS[leg](), "%s: MPMB_NUM_SMS=%d vs unset" % (leg, k))


# ---------------------------------------------------------------------------------------------------- c: oracle files, one SM
ONE_SM_FILES = ["tests/test_gpu_parity.py", "tests/test_gpu_next_p2g.py", "tests/test_gpu_rigid_parity.py", "tests/test_gpu_material_edges.py",
                "tests/test_gpu_slab.py::test_two_slabs_on_one_gpu_match_single_run", "tests/test_gpu_slab.py::test_two_slabs_peer_memory_exchange_one_gpu",
                "tests/test_gpu_slab.py::test_four_slabs_peer_memory_exchange_one_process",
                "tests/test_gpu_slab.py::test_eight_slabs_peer_memory_exchange_one_process",
                "tests/test_gpu_slab_recut.py::test_recut_is_exact_and_the_run_goes_on_like_one_engine",
                "tests/test_gpu_slab_recut.py::test_extreme_cuts_then_substeps_like_one_engine",
                "tests/test_gpu_slab_recut.py::test_append_and_delete_after_a_recut_like_one_engine"]


@pytest.mark.needs_cuda
def test_existing_oracle_files_pass_with_one_sm():
    env = dict(os.environ, MPMB_NUM_SMS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider"] + ONE_SM_FILES,
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


# ---------------------------------------------------------------------------------------------------- d: production grid
def production_scene(seed=13):
    """128^3: about 10 000 active tiles of 8-64 rows and 100 of 600-1200, at rest, 0.4 M particles in all: more tiles
    than k_grid has warps on an H100 (132 x 8 x 8 = 8448), so every kernel walks at least two tiles at its real grid."""
    res = 128
    rng = np.random.default_rng(seed)
    nt = res // 4
    tiles = np.array([(x, y, z) for x in range(2, nt - 2) for y in range(2, nt - 2) for z in range(2, nt - 2)])
    pick = tiles[rng.permutation(len(tiles))[:10100]]
    counts = np.concatenate([rng.integers(600, 1201, 100), rng.integers(8, 65, 10000)])
    X = np.concatenate([rng.uniform(4 * t + 0.55, 4 * t + 4.45, (n, 3)) for t, n in zip(pick, counts)])
    dx = 1.0 / res
    x = (X * dx).astype(np.float32)
    n = len(x)
    vol = np.full(n, dx ** 3 / 8.0, np.float32)
    st = scenes.make_state(x, (vol * np.float32(400.0)).astype(np.float32), vol, scenes.MAT_SAND)
    T.perturb_state(st, scenes.MAT_SAND, dx, seed, vel=0.05)
    scene = dict(res=(res, res, res), dx=dx, dt=2e-5, gravity=(0.0, -10.0, 0.0), particle_gravity=1, clean_boundary=1,
                 mat_kind=np.array([scenes.MAT_SAND], np.int32), mat_params=scenes.material_params(scenes.MAT_SAND)[None],
                 planes=None, friction=0.0, sdf=None)
    return scene, st


@pytest.mark.needs_cuda
def test_production_grid_walks_several_tiles(monkeypatch):
    if SIMT:
        pytest.skip("the production grid is sized for the H100, not for the emulator")
    _hook(monkeypatch, None)
    scene, st = production_scene()
    e = T.make_engine(scene, st)
    worst, states = chain(e, scene, 3, stress=False, all_nodes=False)
    e.close()
    _assert_within(worst, "production grid", TOL_PROD)
    active = [len(np.unique(TS.tile_keys(s["x"], 128))) for s in states]
    assert min(active) > 132 * 8 * 8, active


# ---------------------------------------------------------------------------------------------------- e: bounds-checked build
_CHECKED_SCRIPT = r"""
import json, sys
sys.path.insert(0, %r)
from taichi_mpm_b200 import capi
reports = []
close = capi.Engine.close
def checked_close(self):   # every engine reports its index checks before it goes
    if getattr(self, "h", None) is not None and self.h.value:
        reports.append(self.debug_check())
    close(self)
capi.Engine.close = checked_close
from tests import common as T, tile_shapes as TS, test_gpu_tile_walk as W
scene, st = TS.tile_scene()
e = T.make_engine(scene, st)
worst, states = W.chain(e, scene, TS.NSUB)
e.close()
W._assert_within(worst, "bounds-checked build, MPMB_NUM_SMS=1")
W._assert_guards(states, TS.G2P_CTAS_PER_SM * 3)
W._leg_slabs()
print(json.dumps(reports))
"""


@pytest.mark.needs_cuda
def test_bounds_checked_build_reports_nothing():
    from taichi_mpm_b200 import build
    assert os.path.exists(build.CHECKED_LIB), "the bounds-checked variant is missing: __graft_entry__.build() makes it"
    env = dict(os.environ, MPMB_LIB=build.CHECKED_LIB, MPMB_NUM_SMS="1")
    r = subprocess.run([sys.executable, "-c", _CHECKED_SCRIPT % ROOT], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import json
    reports = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(reports) == 1 + 3 + 3 + 5, reports   # the tile scene; 2, 2 and 4 slabs, each with its one-engine reference
    assert all(rep[0] == 0 for rep in reports), reports
