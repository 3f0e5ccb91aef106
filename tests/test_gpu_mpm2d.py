"""The 2-D engine (MpmbConfig.dim = 2, MPM<2>) against the fp64 2-D oracle (oracle_substep2d), stage by stage, at the
tolerances tests/test_gpu_parity.py applies in 3-D: every material, non-square grids, cell sizes other than 1/res,
two-component gravity, the deletion band and the domain faces with clean_boundary 0 and 1, planes, circles, rectangles
and a dense level set, non-zero dampings, a scene whose particles change cell every substep, a chained run of the
bench_2d.py collapse, CUDA graphs against host launches (bitwise), ids across deletions, the frame writer's records and
the entry points a 2-D handle refuses.  tests/test_mpm2d_simt.py runs this file on the SIMT emulator."""
import os

import numpy as np
import pytest

from taichi_mpm_b200 import capi, scenes
from tests import common as T
from tests.mpm2d_common import perturb2d, scene2d, state_of  # noqa: F401  (also used by tests/test_mpm2d_simt.py)

pytestmark = pytest.mark.gpu

KINDS = [("linear", scenes.MAT_LINEAR), ("jelly", scenes.MAT_JELLY), ("snow", scenes.MAT_SNOW), ("water", scenes.MAT_WATER),
         ("sand", scenes.MAT_SAND), ("elastic", scenes.MAT_ELASTIC), ("von_mises", scenes.MAT_VON_MISES), ("visco", scenes.MAT_VISCO)]


def make_engine2d(scene, st, **kw):
    e = capi.Engine2D(scene["res"], scene["dx"], scene["dt"], scene["gravity"], scene.get("particle_gravity", 1), scene["clean_boundary"],
                      apic_damping=scene.get("apic_damping", 0.0), rpic_damping=scene.get("rpic_damping", 0.0), **kw)
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    route = scene.get("route")
    if route is not None:
        if route[0] == "planes":
            e.set_planes(route[1], scene["friction"])
        elif route[0] == "shapes":
            e.set_levelset_shapes(route[1], scene["friction"])
        else:
            e.set_sdf(scene["sdf"], scene["friction"])
    e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    return e


def compare2d(e, scene, st, check_grid=True, ids=None, yardstick=False, oracle=None):
    """One substep stage by stage on the engine and on the fp64 oracle; the errors as common.compare_substep measures them.
    ids: the engine id of every row of `st` (ascending; default the row index, as after an upload).
    yardstick: also err["yardstick"], the fp32 oracle's errors on the same substep (yardstick2d).
    oracle: the fp64 oracle's substep2d(scene, st) where the caller already has it."""
    from oracle import pyoracle2d as O
    ref, grid_rast, grid_vel = O.substep2d(scene, st, np.float64) if oracle is None else oracle
    e.sort_particles_and_populate_grid()
    e.rasterize()
    grids = (e.download_grid(0), e.download_grid(1)) if check_grid else None
    e.resample()
    got = e.download()
    err = errors2d(got, grids, ref, grid_rast, grid_vel, ids)
    if yardstick:
        err["yardstick"] = yardstick2d(scene, st, ref, grid_rast, grid_vel, ids)
    return err, got, ref


def errors2d(got, grids, ref, grid_rast, grid_vel, ids=None):
    """The errors compare2d reports, of any substep result against the fp64 oracle's: got = dict(id, x, v, b, F, ps, mass) of
    the survivors, grids = (P2G grid, node velocities) or None.  ids: as in compare2d."""
    out = {}
    if grids is not None:
        g0, g1 = (np.asarray(g, np.float64) for g in grids)
        pmax = max(np.abs(grid_rast[..., :2]).max(), grid_rast[..., 3].max())
        out["grid_rast"] = np.abs(g0 - grid_rast).max() / pmax
        m = grid_rast[..., 3]
        active = m > 0
        dv = np.abs(g1[..., :2] - grid_vel[..., :2]).max(-1)
        vmax = max(np.abs(grid_vel[..., :2]).max(), 1e-30)
        out["grid_vel"] = dv[active].max() / vmax
        # the worst node's fp64 mass relative to the heaviest node's, and the same error over the heavy nodes only
        out["grid_vel_node_mass"] = m.flat[np.argmax(np.where(active, dv, -1.0))] / m.max()
        out["grid_vel_heavy"] = dv[m >= HEAVY * m.max()].max() / vmax
        out["grid_mass_outside"] = np.abs(g0[~active]).max() if (~active).any() else 0.0
    alive = ref["alive"].astype(bool)
    row_ids = np.arange(len(alive)) if ids is None else np.asarray(ids, np.int64)
    out["alive_match"] = len(got["id"]) == alive.sum() and np.array_equal(got["id"].astype(np.int64), row_ids[alive])
    if not out["alive_match"] or not alive.any():
        return out
    ids = np.searchsorted(row_ids, got["id"].astype(np.int64))   # oracle row of every downloaded particle
    out["x"] = np.abs(got["x"] - ref["x"][ids]).max()
    out["v"] = np.abs(got["v"] - ref["v"][ids]).max() / np.abs(ref["v"][alive]).max()
    out["b"] = np.abs(got["b"] - ref["b"][ids]).max() / max(np.abs(ref["b"][alive]).max(), 1e-30)
    # F: absolute where |F| <= 1 (tests/common.py), relative above (particles crushed against a face reach |F| ~ 100)
    out["F"] = (np.abs(got["F"] - ref["F"][ids]) / np.maximum(1.0, np.abs(ref["F"][ids]).max(1, keepdims=True))).max()
    out["ps"] = T.ps_err(got["ps"], ref["ps"][ids])
    out["mass"] = np.abs(got["mass"] - ref["mass"][ids]).max()
    return out


def yardstick2d(scene, st, ref, grid_rast, grid_vel, ids=None):
    """The fp32 yardstick: the fp32 oracle's own errors on the same substep of `st`, measured as errors2d measures the engine's
    against the fp64 oracle (ref, grid_rast, grid_vel).  Where the fp32 oracle keeps other survivors (rounding at the band
    edge) its particle errors are not measured and those metrics are held to their tests/common.py bounds alone."""
    from oracle import pyoracle2d as O
    r32, gr32, gv32 = O.substep2d(scene, st, np.float32)
    alive = r32["alive"].astype(bool)
    row_ids = np.arange(len(alive)) if ids is None else np.asarray(ids, np.int64)
    got = {k: r32[k][alive] for k in ("x", "v", "b", "F", "ps", "mass")}
    got["id"] = row_ids[alive]
    return errors2d(got, (gr32, gv32), ref, grid_rast, grid_vel, ids)


# the metrics the yardstick rule applies to and their tests/common.py bounds: the grid, the velocity-normalised ones, and F
# and ps, which G2P forms from the velocity gradient b (cdg = I + dt b (-4 / dx)) and which therefore carry its rounding.
# grid_vel_heavy is grid_vel over the nodes whose fp64 mass is at least HEAVY of the heaviest node's (the 3-D window tests'
# "heavy" nodes): a node whose mass comes only from weights near 0 gets them from the reference's expanded quadratic
# 0.5 t^2 - 1.5 t + 1.125, which fp32 evaluates to about 1e-7 absolute, so its velocity (a weighted mean) is not resolved in
# fp32 and grid_vel there is only held by the yardstick; grid_vel_heavy keeps the node velocities checked on such substeps.
YARD_TOL = dict(grid_rast=T.TOL_GRID_REL, grid_vel=T.TOL_GRID_REL, grid_vel_heavy=T.TOL_GRID_REL, v=T.TOL_V_REL, b=T.TOL_V_REL,
                F=T.TOL_F_ABS, ps=T.TOL_PS_ABS)
YARD_FACTOR = 4.0
HEAVY = 1e-4


def assert_parity_yardstick(err, grid=True, label=""):
    """assert_parity with the yardstick rule on an err of compare2d(..., yardstick=True): a metric of YARD_TOL passes at its
    tests/common.py bound or at YARD_FACTOR times the fp32 oracle's error on the same metric.  Where fp32 itself rounds by
    about that bound (X = x / dx rounded at X ~ 2e3 on a dx that is not a power of two is 6e-5 cells, so dpos, b and cdg of a
    particle moving most of a cell per substep carry it; velocities of 1e-3 m/s in a resting column; hundreds of particles
    summed into one node), the engine is held to what fp32 arithmetic can do rather than to a bound it cannot meet;
    everywhere else the common bound decides.  x keeps its common bound, mass and the mass outside the active nodes stay
    exactly 0, and the survivors are the oracle's."""
    yard = err["yardstick"]
    print(label, {k: "%.3g" % float(v) for k, v in err.items() if k in YARD_TOL or k in ("x", "grid_vel_node_mass")},
          "yardstick", {k: "%.3g" % float(yard[k]) for k in YARD_TOL if k in yard})
    assert err["alive_match"], (label, err)
    for k, tol in YARD_TOL.items():
        if k in err and (grid or not k.startswith("grid")):
            assert err[k] <= tol or err[k] <= YARD_FACTOR * yard.get(k, 0.0), (label, k, err[k], tol, yard.get(k))
    if grid:
        assert err["grid_mass_outside"] == 0.0, (label, err)
    assert err["x"] <= T.TOL_X_ABS, (label, err)
    assert err["mass"] == 0.0, (label, err)


def assert_parity(err, grid=True):
    assert err["alive_match"], err
    if grid:
        assert err["grid_rast"] <= T.TOL_GRID_REL, err
        assert err["grid_vel"] <= T.TOL_GRID_REL, err
        assert err["grid_mass_outside"] == 0.0, err
    assert err["x"] <= T.TOL_X_ABS, err
    assert err["v"] <= T.TOL_V_REL, err
    assert err["b"] <= T.TOL_V_REL, err
    assert err["F"] <= T.TOL_F_ABS, err
    assert err["ps"] <= T.TOL_PS_ABS, err
    assert err["mass"] == 0.0, err


@pytest.mark.parametrize("name,kind", KINDS, ids=[k[0] for k in KINDS])
def test_every_material_one_substep(name, kind):
    kw = dict(strain=0.006) if kind == scenes.MAT_VON_MISES else {}
    if kind == scenes.MAT_VISCO:
        kw["kappa"] = 0.3
    scene, st = scene2d(kind, seed=1, **kw)
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st)
    assert_parity(err)
    e.close()


@pytest.mark.parametrize("name,kind", KINDS, ids=[k[0] for k in KINDS])
def test_every_material_chained_substeps(name, kind):
    """10 substeps, each one compared: the engine's state after k substeps is the oracle's input for substep k + 1."""
    scene, st = scene2d(kind, seed=2, vel=0.3)
    e = make_engine2d(scene, st)
    for _ in range(10):
        now = e.download()
        err, _, _ = compare2d(e, scene, state_of(now), check_grid=False, ids=now["id"])
        assert_parity(err, grid=False)
    e.close()


# non-square grids: res + 1 takes every remainder modulo the 16-node tile edge across the cases (17 % 16 = 1 ... 32 % 16 = 0)
GRIDS = [((16 + k, 48 - k), 1.0 / (16 + k) * (0.9 + 0.02 * k)) for k in range(16)]


@pytest.mark.parametrize("res,dx", GRIDS, ids=["%dx%d" % r for r, _ in GRIDS])
def test_non_square_grids(res, dx):
    lo = (res[0] // 2 - 2, 8)
    scene, st = scene2d(scenes.MAT_JELLY, res=res, dx=dx, blocks=[(lo, (lo[0] + 4, lo[1] + 6))], gravity=(3.0, -8.0), seed=3)
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st)
    assert_parity(err)
    e.close()


@pytest.mark.parametrize("clean", [1, 0])
def test_band_and_domain_faces(clean):
    """Particles in the 7-cell band and next to every face, moving outwards: the band deletes with clean_boundary = 1; with
    clean_boundary = 0 the position clamp and the off-grid rule do."""
    res = (32, 40)
    blocks = [((1, 10), (4, 14)), ((28, 10), (32, 14)), ((10, 0), (14, 4)), ((10, 36), (14, 40)), ((6, 20), (9, 24)), ((14, 14), (18, 18))]
    scene, st = scene2d(scenes.MAT_JELLY, res=res, blocks=blocks, levelset=None, clean_boundary=clean, seed=4, jitter=0.24, vel=0.0)
    c = np.array([16, 20], np.float32) / res[0]
    st["v"] = ((st["x"] - c) * 400.0).astype(np.float32)   # outwards, about half a cell per substep near the faces
    st["x"][0] = [0.3 / res[0], 12.2 / res[0]]             # within half a cell of the lower face: int(X - 0.5) = 0
    e = make_engine2d(scene, st)
    for k in range(3):
        now = e.download()
        err, got, ref = compare2d(e, scene, st if k == 0 else state_of(now), check_grid=(k == 0), ids=None if k == 0 else now["id"])
        assert_parity(err, grid=(k == 0))
        if k == 0:
            assert 0 < ref["alive"].sum() < len(st["x"])
    assert (got["x"] * res[0] <= np.array(res, np.float32)).all() and (got["x"] >= 0).all()
    e.close()


@pytest.mark.parametrize("friction", [-1.0, -2.0, -2.3, 0.0, 0.4])
@pytest.mark.parametrize("clean", [1, 0])
def test_plane_boundary_modes(friction, clean):
    scene, st = scene2d(scenes.MAT_JELLY, seed=5, friction=friction, clean_boundary=clean, vel=1.0)
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st)
    assert_parity(err)
    e.close()


LEVELSETS = {
    "planes": ("planes", [[0.0, 1.0, 0.0, -9.6], [0.7071067811865476, 0.7071067811865476, 0.0, -25.0]]),
    "circle": ("shapes", [(1, 0, (16.0, 6.0, 0.0, 3.4))]),
    "container": ("shapes", [(1, 1, (16.0, 14.0, 0.0, 9.0))]),
    "rectangle": ("shapes", [(2, 0, (10.0, 4.0, 0.0, 22.0, 9.6, 0.0)), (0, 0, (1.0, 0.0, 0.0, -10.0))]),
    "dense": ("dense", [(2, 1, (8.0, 9.5, 0.0, 24.0, 30.0, 0.0)), (1, 0, (16.0, 9.0, 0.0, 2.0))]),
}


@pytest.mark.parametrize("name", sorted(LEVELSETS))
def test_level_sets(name):
    scene, st = scene2d(scenes.MAT_SAND, seed=6, levelset=LEVELSETS[name], friction=0.3, vel=1.0)
    phi = scene["sdf"][..., 3]
    assert (phi <= 0).any() and (phi > 0).any() and (np.abs(phi) < 3).any()
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st)
    assert_parity(err)
    e.close()


def test_shapes_with_a_z_part_are_refused():
    scene, st = scene2d(scenes.MAT_JELLY, seed=7, levelset=None)
    e = make_engine2d(scene, st)
    for shapes in ([(1, 0, (16.0, 6.0, 1.0, 3.0))], [(2, 0, (1.0, 1.0, 0.0, 5.0, 5.0, 2.0))], [(0, 0, (0.0, 0.8, 0.6, -3.0))]):
        with pytest.raises(capi.MpmbError):
            e.set_levelset_shapes(shapes, 0.0)
    e.close()


@pytest.mark.parametrize("apic,rpic", [(0.3, 0.0), (0.0, 0.5), (1.0, 0.25)])
def test_dampings(apic, rpic):
    scene, st = scene2d(scenes.MAT_JELLY, seed=8, apic=apic, rpic=rpic)
    e = make_engine2d(scene, st)
    err, got, ref = compare2d(e, scene, st)
    assert_parity(err)
    b = got["b"].reshape(-1, 2, 2).transpose(0, 2, 1)
    if apic == 1.0:   # the skew part is gone
        assert np.abs(b - b.transpose(0, 2, 1)).max() <= 1e-6 * np.abs(b).max()
    e.close()


def test_grid_gravity_and_two_materials():
    sc1, st1 = scene2d(scenes.MAT_SAND, seed=9, particle_gravity=0, gravity=(2.0, -9.0))
    x2, m2, v2 = scenes.lattice_block2d((32, 32), (10, 20), (14, 24), dx=sc1["dx"])
    st2 = scenes.make_state2d(x2, m2, v2, scenes.MAT_WATER, group=1)
    st = {k: np.concatenate([st1[k], st2[k]]) for k in st1}
    scene = dict(sc1, mat_kind=np.array([scenes.MAT_SAND, scenes.MAT_WATER], np.int32),
                 mat_params=np.stack([scenes.material_params(scenes.MAT_SAND), scenes.material_params(scenes.MAT_WATER)]))
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st)
    assert_parity(err)
    e.close()


def test_particles_change_cell_every_substep():
    """A fast shear flow over many node tiles: most particles leave their cell each substep, the ordering re-bins them."""
    res = (80, 72)
    scene, st = scene2d(scenes.MAT_WATER, res=res, blocks=[((8, 8), (72, 64))], levelset=None, seed=10, vel=0.0, jitter=0.2, dt=2e-4)
    X = st["x"] * res[0]
    # up to 0.9 cells per substep
    st["v"] = (np.stack([np.sin(X[:, 1] * 0.3), np.cos(X[:, 0] * 0.2)], 1) * 0.9 / res[0] / 2e-4).astype(np.float32)
    e = make_engine2d(scene, st)
    moved = 0.0
    for k in range(3):
        before = e.download()
        err, got, ref = compare2d(e, scene, st if k == 0 else state_of(before), check_grid=(k == 0), ids=None if k == 0 else before["id"])
        assert_parity(err, grid=(k == 0))
        keep = np.isin(before["id"], got["id"])
        cb = np.floor(before["x"][keep] * res[0] - 0.5).astype(int)
        ca = np.floor(got["x"] * res[0] - 0.5).astype(int)
        moved = max(moved, (cb != ca).any(1).mean())
    assert moved > 0.4, moved
    e.close()


def crowded_state(scene, lo, hi, ppc, seed):
    """n x n particles per cell (ppc = n^2) over cells [lo, hi), jittered within their sub-cells, vol = dx^2 / ppc and mass
    400 vol (the density of the 4-per-cell lattice), perturbed as scene2d perturbs its blocks."""
    dx, n = scene["dx"], int(round(np.sqrt(ppc)))
    rng = np.random.default_rng(seed)
    c = np.stack(np.meshgrid(np.arange(lo[0], hi[0]), np.arange(lo[1], hi[1]), indexing="ij"), -1).reshape(-1, 1, 2)
    s = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(1, -1, 2)
    X = (c + (s + 0.5 + rng.uniform(-0.3, 0.3, (c.shape[0], s.shape[1], 2))) / n).reshape(-1, 2)
    vol = np.full(len(X), dx * dx / ppc, np.float32)
    st = scenes.make_state2d((X * dx).astype(np.float32), vol * np.float32(400.0), vol, scenes.MAT_SAND)
    return perturb2d(st, scenes.MAT_SAND, dx, seed)


# particles per cell and cells per side: the developed column reaches 6 to 8 per cell (DESIGN §10); k2_grid sums every
# particle of a node's 3 x 3 cells in one fixed-order fp32 loop, so its rounding grows with the count.  Measured on an
# NVIDIA H100 80GB HBM3 (700 W power limit), grid_rast / grid_vel / v / b / F / ps: 16: 5.1e-7 / 4.2e-7 / 4.4e-7 / 7.3e-6 /
# 2.9e-7 / 2.7e-7; 64: 7.5e-7 / 6.3e-7 / 6.8e-7 / 9.8e-6 / 3.4e-7 / 2.5e-7; 256: 7.7e-7 / 1.7e-6 / 1.4e-6 / 2.0e-5 / 3.5e-7 /
# 3.1e-7; 4096 in one cell: 9.7e-7 / 2.1e-6 / 9.8e-7 / 3.7e-5 / 3.6e-7 / 2.9e-7; test_stencil_base_switch: 1.6e-7 / 1.6e-7 /
# 1.4e-7 / 3.1e-6 / 2.3e-7 / 2.3e-7.  All are inside the tests/common.py bounds: the yardstick rule passes none of them.
CROWDED = {"16": (16, 8), "64": (64, 6), "256": (256, 4), "4096_in_one_cell": (4096, 1)}


@pytest.mark.parametrize("name", list(CROWDED))
def test_crowded_cells(name):
    ppc, cells = CROWDED[name]
    lo = (14, 10)
    hi = (lo[0] + cells, lo[1] + cells)
    scene, _ = scene2d(scenes.MAT_SAND, blocks=[(lo, hi)], seed=30)
    st = crowded_state(scene, lo, hi, ppc, seed=31)
    cell = np.floor(st["x"].astype(np.float64) / scene["dx"]).astype(int)
    assert np.unique(cell[:, 0] * 64 + cell[:, 1], return_counts=True)[1].min() == ppc
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st, yardstick=True)
    assert_parity_yardstick(err, label="crowded %s" % name)
    e.close()


def test_stencil_base_switch():
    """Particles exactly at X = k and X = k + 0.5 on each axis (dx = 2^-5, so X is exact in fp32): at X = k + 0.5 the stencil
    base int(X - 0.5) switches to k and the fraction is 0, at X = k the base is k - 1 and the fraction 1/2."""
    lo, hi = (12, 10), (20, 18)
    scene, _ = scene2d(scenes.MAT_SAND, blocks=[(lo, hi)], seed=32)
    X = np.stack(np.meshgrid(np.arange(2 * lo[0], 2 * hi[0]) * 0.5, np.arange(2 * lo[1], 2 * hi[1]) * 0.5, indexing="ij"), -1).reshape(-1, 2)
    vol = np.full(len(X), scene["dx"] ** 2 / 4, np.float32)
    st = perturb2d(scenes.make_state2d((X * scene["dx"]).astype(np.float32), vol * np.float32(400.0), vol, scenes.MAT_SAND),
                   scenes.MAT_SAND, scene["dx"], 33)
    assert np.array_equal(st["x"].astype(np.float64) / scene["dx"], X)
    e = make_engine2d(scene, st)
    err, _, _ = compare2d(e, scene, st, yardstick=True)
    assert_parity_yardstick(err, label="stencil base switch")
    e.close()


def test_graph_replay_is_bitwise_equal_to_host_launches():
    scene, st = scene2d(scenes.MAT_SAND, seed=11, vel=0.5)
    outs = []
    for no_graph in (False, True):
        e = make_engine2d(scene, st, no_graph=no_graph)
        e.substep(5)
        e.substep(4)
        outs.append(e.download())
        assert e.update_count() == 9 * len(st["x"]) or e.num_particles() < len(st["x"])
        e.close()
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), k


def test_ids_survive_substeps_and_deletions():
    scene, st = scene2d(scenes.MAT_JELLY, seed=12, levelset=None, vel=0.0)
    st["x"][3] = [7.2 / 32, 0.5]
    st["v"][3] = [-300.0, 0.0]     # into the band: deleted by the first G2P
    e = make_engine2d(scene, st)
    e.set_id_base(1000)
    e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    e.substep(4)
    got = e.download()
    assert 1003 not in got["id"] and len(got["id"]) == len(st["x"]) - 1 == e.num_particles()
    assert np.array_equal(got["id"], np.setdiff1d(np.arange(1000, 1000 + len(st["x"])), [1003]))
    # each particle is still the one it was: its mass and volume travel with the id
    assert np.array_equal(got["mass"], np.delete(st["mass"], 3)) and np.array_equal(got["vol"], np.delete(st["vol"], 3))
    assert e.update_count() == len(st["x"]) + 3 * (len(st["x"]) - 1)
    e.close()


def test_bgeo_records_in_id_order_with_zero_third_components():
    scene, st = scene2d(scenes.MAT_JELLY, seed=13)
    e = make_engine2d(scene, st)
    e.substep(2)
    n, rec = e.download_bgeo_points(len(st["x"]))
    got = e.download()
    assert n == len(got["id"])
    w = rec.view(">u4").reshape(n, 12)
    f = rec.view(">f4").reshape(n, 12)
    assert np.array_equal(w[:, 5], got["id"]) and (w[:, 4] == 0).all() and (w[:, 6:9] == 1).all()
    assert np.array_equal(f[:, 0:2], got["x"]) and (w[:, 2] == 0).all() and (f[:, 3] == 1.0).all()
    assert np.array_equal(f[:, 9:11], got["v"]) and (w[:, 11] == 0).all()
    e.close()


def test_collapse_chained_against_the_chained_oracle():
    """bench_2d.py's sand column at reduced size (64^2 grid, 32x32-cell column, 4 per cell), 200 substeps on both sides from
    the same state: same survivors, centre of mass and momentum; then one substep compared stage by stage from there."""
    from oracle import pyoracle2d as O
    res, cells = 64, 32
    scene, st = scene2d(scenes.MAT_SAND, res=(res, res), blocks=[((16, 8), (16 + cells, 8 + cells))], levelset=("planes", [[0.0, 1.0, 0.0, -8.0]]),
                        friction=0.4, dt=2e-5 * 1024 / res / 4, seed=14, vel=0.0, jitter=0.0, strain=0.0)
    st["ps"][:] = 0.0
    st["b"][:] = 0.0
    e = make_engine2d(scene, st)
    ref = st
    for _ in range(200):
        ref = O.substep2d(scene, ref, np.float64, want_grids=False)[0]
    e.substep(200)
    got = e.download()
    alive = ref["alive"].astype(bool)
    assert np.array_equal(got["id"], np.nonzero(alive)[0])
    m = got["mass"].astype(np.float64)
    com_g, com_o = (m[:, None] * got["x"]).sum(0) / m.sum(), (m[:, None] * ref["x"][alive]).sum(0) / m.sum()
    mom_g, mom_o = (m[:, None] * got["v"]).sum(0), (m[:, None] * ref["v"][alive]).sum(0)
    assert np.abs(com_g - com_o).max() < 2e-5
    assert np.abs(mom_g - mom_o).max() <= 2e-3 * max(np.abs(mom_o).max(), m.sum() * 0.01)
    assert np.abs(got["v"]).max() > 0.01   # the column is moving
    err, _, _ = compare2d(e, scene, state_of(got), ids=got["id"])
    assert_parity(err)
    e.close()


def test_refused_entry_points():
    scene, st = scene2d(scenes.MAT_JELLY, seed=15)
    e = make_engine2d(scene, st)
    L, h = e.L, e.h
    n = capi.C.c_int64(0)
    calls = {
        "append_particles": lambda: L.mpmb_append_particles(h, 0, None, None, None, None, None, None, None, None, None),
        "append_owned_particles": lambda: L.mpmb_append_owned_particles(h, 0, None, None, None, None, None, None, None, None, 0, capi.C.byref(n)),
        "delete_inside_levelset": lambda: L.mpmb_delete_inside_levelset(h, capi.C.byref(n)),
        "delete_owned_inside_levelset": lambda: L.mpmb_delete_owned_inside_levelset(h, capi.C.byref(n)),
        "id_end": lambda: L.mpmb_id_end(h, capi.C.byref(n)),
        "upload_aos": lambda: L.mpmb_upload_aos(h, 0, None, 0, None, None, None),
        "download_aos": lambda: L.mpmb_download_aos(h, None, 0, None, 0, None, None),
        "seed_lattice": lambda: L.mpmb_seed_lattice(h, None, None, capi.C.c_float(1), capi.C.c_float(1), capi.C.c_float(0), 0, 0, None, None),
        "set_rigid_samples": lambda: L.mpmb_set_rigid_samples(h, 0, 0, None, None, None),
        "set_rigid_coupling": lambda: L.mpmb_set_rigid_coupling(h, capi.C.c_float(0), capi.C.c_float(0)),
        "set_rigid_state": lambda: L.mpmb_set_rigid_state(h, 0, None),
        "get_rigid_state": lambda: L.mpmb_get_rigid_state(h, 0, None),
        "set_rigid_motion": lambda: L.mpmb_set_rigid_motion(h, 0, None, 0),
        "set_rigid_script": lambda: L.mpmb_set_rigid_script(h, 0, None),
        "set_particle_states": lambda: L.mpmb_set_particle_states(h, 0, None),
        "get_particle_cdf": lambda: L.mpmb_get_particle_cdf(h, 0, None, None, None, None),
        "download_cdf": lambda: L.mpmb_download_cdf(h, None, None),
        "rasterize_part": lambda: L.mpmb_rasterize_part(h, 1),
        "resample_part": lambda: L.mpmb_resample_part(h, 1),
        "get_ordering_stats": lambda: L.mpmb_get_ordering_stats(h, None, None, None),
        "halo_bytes": lambda: L.mpmb_halo_bytes(h),
        "halo_pack": lambda: L.mpmb_halo_pack(h, 0, None),
        "halo_unpack": lambda: L.mpmb_halo_unpack(h, 0, None),
        "migrate_bytes": lambda: L.mpmb_migrate_bytes(h),
        "migrate_pack": lambda: L.mpmb_migrate_pack(h, 0, None),
        "migrate_unpack": lambda: L.mpmb_migrate_unpack(h, 0, None),
        "xchg_buffer": lambda: L.mpmb_xchg_buffer(h, 0, 0, None),
        "xchg_ipc_handle": lambda: L.mpmb_xchg_ipc_handle(h, 0, 0, None),
        "xchg_connect": lambda: L.mpmb_xchg_connect(h, 0, 0, None, None),
        "halo_send": lambda: L.mpmb_halo_send(h, 0),
        "halo_recv": lambda: L.mpmb_halo_recv(h, 0),
        "migrate_send": lambda: L.mpmb_migrate_send(h, 0),
        "migrate_recv": lambda: L.mpmb_migrate_recv(h, 0),
        "layer_counts": lambda: L.mpmb_layer_counts(h, 0, None),
        "recut_pack": lambda: L.mpmb_recut_pack(h, None, None, 0, None),
        "recut_apply": lambda: L.mpmb_recut_apply(h, 0, 1, 0, None),
        "rigid_impulse_bytes": lambda: L.mpmb_rigid_impulse_bytes(h),
        "rigid_impulse_pack": lambda: L.mpmb_rigid_impulse_pack(h, None),
        "rigid_impulse_apply": lambda: L.mpmb_rigid_impulse_apply(h, None),
        "rigid_mailbox": lambda: L.mpmb_rigid_mailbox(h, None),
        "rigid_mailbox_ipc_handle": lambda: L.mpmb_rigid_mailbox_ipc_handle(h, None),
        "rigid_connect": lambda: L.mpmb_rigid_connect(h, 1, None, None),
        "rigid_send": lambda: L.mpmb_rigid_send(h),
        "rigid_recv": lambda: L.mpmb_rigid_recv(h),
        "async_init": lambda: L.mpmb_async_init(h, None, capi.C.c_float(1)),
        "async_add": lambda: L.mpmb_async_add(h, 0, 0, None, None, None, None, None, None, None, None, None),
        "async_block_limits": lambda: L.mpmb_async_block_limits(h, 0, 0, None, None, None, None),
        "async_advance": lambda: L.mpmb_async_advance(h, None, capi.C.c_float(1e-4), None),
        "async_size": lambda: L.mpmb_async_size(h, None, None),
        "async_download": lambda: L.mpmb_async_download(h, 0, 0, None, None, None, None, None, None, None, None, None, None, None),
        "async_schedule": lambda: L.mpmb_async_schedule(h, 0, capi.C.c_float(1), capi.C.c_float(1), capi.C.c_float(1), capi.C.c_float(1), 1, None, None),
        "async_advance_level": lambda: L.mpmb_async_advance_level(h, 0, 1, capi.C.c_float(1e-4), None),
        "async_block_state": lambda: L.mpmb_async_block_state(h, None, None, None, None),
    }
    assert set("mpmb_" + k for k in calls) | {"mpmb_create", "mpmb_destroy", "mpmb_last_error", "mpmb_version", "mpmb_set_stream",
                                              "mpmb_synchronize", "mpmb_set_material", "mpmb_set_delta_t", "mpmb_set_sdf", "mpmb_set_planes",
                                              "mpmb_set_levelset_shapes", "mpmb_set_id_base", "mpmb_upload_particles", "mpmb_num_particles",
                                              "mpmb_get_update_count", "mpmb_download_bgeo_points", "mpmb_download_particles", "mpmb_substep",
                                              "mpmb_sort_particles_and_populate_grid", "mpmb_rasterize", "mpmb_resample",
                                              "mpmb_download_grid", "mpmb_set_profiling", "mpmb_get_profile", "mpmb_get_counters"} == set(capi.EXPORTS)
    for name, call in calls.items():
        rc = call()
        assert rc < 0, name
        assert b"2-D handle" in L.mpmb_last_error(h), name
    # the handle is still usable
    e.substep(2)
    assert e.num_particles() == len(st["x"])
    e.close()


def test_create_checks_the_2d_config():
    with pytest.raises(capi.MpmbError):   # dampings are MPM<2> only
        capi.Engine((32, 32, 32), 1 / 32, 1e-4, apic_damping=0.5)
    with pytest.raises(capi.MpmbError):   # a z extent on a 2-D handle
        capi.Engine((32, 32, 32), 1 / 32, 1e-4, dim=2)
    with pytest.raises(capi.MpmbError):   # gravity along z
        capi.Engine((32, 32), 1 / 32, 1e-4, gravity=(0.0, -10.0, 1.0), dim=2)
    with pytest.raises(capi.MpmbError):
        capi.Engine((32, 32, 32), 1 / 32, 1e-4, dim=4)


def test_profile_and_counters():
    scene, st = scene2d(scenes.MAT_SAND, seed=16)
    e = make_engine2d(scene, st)
    e.set_profiling(True)
    e.substep(3)
    ms, launches = e.get_profile()
    assert launches[0] == 9 and launches[1] == 6 and launches[2] == 3, launches
    if not os.environ.get("MPMB_SIMT"):
        assert all(t > 0 for t in ms[:3]), ms
    c = e.get_counters()
    assert c["alive"] == len(st["x"]) and c["active_tiles"] == 9 and c["kernel_launches"] > 0
    e.close()


def _golden_maker():
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_mpm2d_golden.py")
    spec = importlib.util.spec_from_file_location("make_mpm2d_golden", path)
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


@pytest.mark.parametrize("name,kind", KINDS, ids=[k[0] for k in KINDS])
def test_engine_matches_golden_run_of_reference_substeps(name, kind):
    """The reference's own MPM<2>::substep(), 12 substeps recorded in tests/golden/mpm2d_ref.npz (two particles start in the
    band), against the engine from the same state, at the bounds tests/test_gpu_zz_reference_golden.py applies in 3-D."""
    G = _golden_maker()
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mpm2d_ref.npz"))
    scene, st = G.substep_scene(kind)
    e = make_engine2d(scene, st)
    e.substep(G.SUBSTEPS)
    got = e.download()
    alive = z["k%d_sub_alive" % kind].astype(bool)
    assert np.array_equal(got["id"], np.nonzero(alive)[0])
    ref = {k: z["k%d_sub_%s" % (kind, k)][alive] for k in ("x", "v", "F", "b", "ps")}
    assert np.abs(got["x"] - ref["x"]).max() <= 1e-5
    assert np.abs(got["v"] - ref["v"]).max() <= 1e-3 * np.abs(ref["v"]).max()
    assert np.abs(got["b"] - ref["b"]).max() <= 2e-3 * np.abs(ref["b"]).max()
    if kind != scenes.MAT_WATER:
        assert np.abs(got["F"] - ref["F"]).max() <= 2e-4
    assert T.ps_err(got["ps"], ref["ps"]) <= (1e-3 if kind == scenes.MAT_VISCO else 1e-4)
    e.close()


def test_bgeo_points_are_the_bytes_of_the_reference_writer(tmp_path):
    """tests/golden/frame2d_ref.bgeo is MPM<2>::write_partio's frame (src/visualize.cpp:16-100, through the vendored Partio):
    its particles uploaded to the engine come back through mpmb_download_bgeo_points + bgeo.write_bgeo_packed as the same
    file, byte for byte (z and v_z are 0, as the dim loops of the writer leave them)."""
    from taichi_mpm_b200 import bgeo
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame2d_ref.bgeo")
    pos, attrs = bgeo.read_bgeo(golden)
    a = {name: arr for name, _, arr in attrs}
    n = len(pos)
    assert (pos[:, 2] == 0).all() and (a["v"].reshape(n, 3)[:, 2] == 0).all()
    assert np.array_equal(a["index"].ravel(), np.arange(n))
    G = _golden_maker()
    scene, st = G.golden_scene(scenes.MAT_SAND)
    e = make_engine2d(scene, st)
    e.upload(pos[:, :2], a["v"].reshape(n, 3)[:, :2], st["mass"][:n], st["vol"][:n])
    k, block = e.download_bgeo_points(n)
    out = str(tmp_path / "frame.bgeo")
    bgeo.write_bgeo_packed(out, k, block)
    assert open(out, "rb").read() == open(golden, "rb").read()
    e.close()


def test_empty_and_single_particle_sets():
    scene, st = scene2d(scenes.MAT_JELLY, seed=17)
    one = {k: v[:1] for k, v in st.items()}
    e = make_engine2d(scene, one)
    err, _, _ = compare2d(e, scene, one)
    assert_parity(err)
    e.close()
    e = capi.Engine2D(scene["res"], scene["dx"], scene["dt"])
    e.upload(np.zeros((0, 2)), np.zeros((0, 2)), np.zeros(0), np.zeros(0))
    e.substep(3)
    assert e.num_particles() == 0 and len(e.download()["id"]) == 0 and e.update_count() == 0
    e.close()
