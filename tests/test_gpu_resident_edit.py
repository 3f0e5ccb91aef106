"""Edits of the resident particle set on the device: mpmb_append_particles (MPM<3>::add_particles mid-run, src/mpm.cpp:147)
and mpmb_delete_inside_levelset (delete_particles_inside_level_set, src/mpm.cpp:959-973).  Resident particles keep their
rows' state, ids and CPIC colours; new particles are numbered after every id handed out so far.  Runs on the SIMT emulator
too (tests/test_resident_edit_simt.py)."""
import numpy as np
import pytest

from taichi_mpm_b200 import capi, mpm as mpm_mod, scenes
from tests import common as T
from tests.test_gpu_parity import _assert_parity

pytestmark = pytest.mark.gpu

FIELDS = ("x", "v", "F", "b", "mass", "vol", "ps", "group")
OUT = ("id", "x", "v", "F", "b", "mass", "vol", "ps", "group")


def _take(st, sel):
    return {k: np.ascontiguousarray(st[k][sel]) for k in FIELDS}


def _cat(a, b):
    return {k: np.concatenate([a[k], b[k]]) for k in FIELDS}


def _append(e, s):
    return e.append(s["x"], s["v"], s["mass"], s["vol"], s["F"], s["b"], s["ps"], s["group"])


def _as_state(d):
    st = {k: np.ascontiguousarray(d[k]) for k in FIELDS}
    st["alive"] = np.ones(len(st["x"]), np.uint8)
    return st


def _bare_engine(scene, **kw):
    """T.make_engine without the upload."""
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], scene.get("particle_gravity", 1), scene.get("clean_boundary", True), **kw)
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    if scene.get("planes") is not None:
        e.set_planes(scene["planes"], scene["friction"])
    return e


def _movers_scene(kind):
    """Two blocks moving towards each other across tile faces on all three axes; the second block is the one appended."""
    res, dx = (40, 34, 44), 1.0 / 33
    scene, st = T.general_scene(kind, res, dx, [((10, 9, 10), (16, 13, 16)), ((22, 10, 24), (28, 14, 30))], (0.0, -10.0, 0.0),
                                levelset=("planes", np.array([[0.05, 1.0, -0.03, -8.6]], np.float32)), dt=1e-4,
                                strain=0.01 if kind == scenes.MAT_SAND else 0.02, vel=0.0, seed=23)
    x = st["x"] / np.float32(scene["dx"])
    c = x.mean(0)
    rng = np.random.default_rng(24)
    n = len(x)
    st["v"] = np.stack([np.where(x[:, 0] < c[0], 2.5, -2.5), np.full(n, 1.5), np.where(x[:, 2] < c[2], 2.0, -2.0)], 1)
    st["v"] = (st["v"] + 0.2 * rng.normal(size=(n, 3))).astype(np.float32)
    second = x[:, 0] > c[0]
    return scene, _take(st, ~second), _take(st, second)


def _assert_same(a, b, keys=OUT):
    assert len(a["id"]) == len(b["id"])
    for k in keys:
        assert np.array_equal(a[k], b[k]), k


def test_append_keeps_the_resident_rows_and_numbers_new_ids_after_the_span():
    scene, s1, s2 = _movers_scene(scenes.MAT_JELLY)
    e = T.make_engine(scene, s1)
    e.substep(5)
    a = e.download()
    first = _append(e, s2)
    b = e.download()
    e.close()
    n1, n2 = len(s1["x"]), len(s2["x"])
    assert first == n1 and len(a["id"]) == n1
    assert len(b["id"]) == n1 + n2 and np.array_equal(b["id"], np.arange(n1 + n2))
    _assert_same({k: v[:n1] for k, v in b.items()}, a)                          # A's rows and ids: bit for bit
    for k in FIELDS:                                                               # S2 with ids first .. first + n2 - 1
        assert np.array_equal(b[k][n1:], s2[k]), k
    # after seeding, the new ids continue after the lattice's id range, not after the number of seeded particles
    e = _bare_engine(scene)
    vol = np.float32(scene["dx"]) ** 3 / 8
    n_seeded = e.seed_lattice((4, 10, 10), (12, 14, 14), vol, vol * 400)
    lattice = 8 * 4 * 4 * 8
    assert 0 < n_seeded < lattice                                                  # cells 4..6 lie in the 7-cell band
    assert _append(e, s2) == lattice
    d = e.download()
    assert np.array_equal(d["id"][-n2:], np.arange(lattice, lattice + n2)) and len(d["id"]) == n_seeded + n2
    e.close()


@pytest.mark.parametrize("kind", [scenes.MAT_JELLY, scenes.MAT_SAND], ids=["jelly", "sand"])
def test_substeps_after_an_append_follow_the_oracles(kind):
    from oracle import pyoracle as O
    scene, s1, s2 = _movers_scene(kind)

    def edited():
        e = T.make_engine(scene, s1)
        e.substep(3)
        _append(e, s2)
        return e

    e = edited()
    union = e.download()
    assert np.array_equal(union["id"], np.arange(len(union["id"])))            # ids == rows of the oracle's state
    u = _as_state(union)
    err, _, _ = T.compare_substep(e, scene, u)
    e.close()
    _assert_parity(err)
    nsub = 24
    fast = O.FastOracle(scene, u, threads=4)
    fast.substeps(nsub)
    e = edited()
    e.substep(nsub)
    got = e.download()
    e.close()
    tile = lambda x: (x * (np.float32(1) / np.float32(scene["dx"])) - np.float32(0.5)).astype(np.int32) >> 2
    tb0, tb1 = tile(u["x"][got["id"]]), tile(got["x"])
    assert all((tb0[:, d] != tb1[:, d]).sum() > 20 for d in range(3))            # particles crossed tile faces on every axis
    alive = fast.st["alive"].astype(bool)
    ids = got["id"].astype(np.int64)
    assert np.array_equal(ids, np.nonzero(alive)[0])
    assert np.abs(got["x"] - fast.st["x"][ids]).max() < 5e-5
    assert np.abs(got["v"] - fast.st["v"][ids]).max() < 2e-2 * np.abs(fast.st["v"]).max()


def test_graph_replay_and_host_launches_agree_across_an_append_and_runs_repeat():
    scene, s1, s2 = _movers_scene(scenes.MAT_SAND)
    outs = []
    for no_graph in (False, True, False):
        e = T.make_engine(scene, s1, no_graph=no_graph)
        e.substep(7)
        _append(e, s2)
        e.substep(9)
        outs.append(e.download())
        e.close()
    _assert_same(outs[0], outs[1])
    _assert_same(outs[0], outs[2])


def test_growing_on_append_equals_a_large_fixed_capacity_and_a_small_one_is_refused():
    scene, s1, s2 = _movers_scene(scenes.MAT_SAND)
    n1, n2 = len(s1["x"]), len(s2["x"])
    outs = []
    for cap in (0, 10 * (n1 + n2)):
        e = T.make_engine(scene, s1, capacity=cap)
        e.substep(4)
        _append(e, s2)
        _append(e, _take(s2, slice(0, 7)))                       # a second append, onto the grown buffers
        e.substep(6)
        outs.append(e.download())
        e.close()
    _assert_same(outs[0], outs[1])
    e = T.make_engine(scene, s1, capacity=n1 + n2 // 2)
    ref = T.make_engine(scene, s1)
    e.substep(4); ref.substep(4)
    before = e.download()
    with pytest.raises(capi.MpmbError) as ex:
        _append(e, s2)
    assert ex.value.code == -3                                   # MPMB_ERR_CAPACITY
    _assert_same(e.download(), before)
    e.substep(6); ref.substep(6)
    _assert_same(e.download(), ref.download())
    assert _append(e, _take(s2, slice(0, 3))) == n1              # a refused append hands out no ids
    e.close(); ref.close()


def test_append_onto_an_empty_engine_or_right_after_an_upload_equals_one_upload():
    scene, s1, s2 = _movers_scene(scenes.MAT_JELLY)
    u = _cat(s1, s2)
    ref = T.make_engine(scene, u)
    ref.substep(10)
    want = ref.download()
    ref.close()
    e = _bare_engine(scene)                                      # never uploaded
    assert _append(e, u) == 0
    e.substep(10)
    _assert_same(e.download(), want)
    e.close()
    e = T.make_engine(scene, s1)                                 # before any substep
    before = e.download()
    assert _append(e, _take(s2, slice(0, 0))) == len(s1["x"])   # n = 0: nothing changes
    _assert_same(e.download(), before)
    assert _append(e, s2) == len(s1["x"])
    e.substep(10)
    _assert_same(e.download(), want)
    e.close()


def test_append_drops_non_finite_and_out_of_grid_particles_as_an_upload_does():
    scene, s1, s2 = _movers_scene(scenes.MAT_JELLY)
    bad = _take(s2, slice(0, 8))
    bad["x"][0, 0] = np.nan
    bad["x"][1, 1] = np.inf
    bad["x"][2] = (-0.01, 0.5, 0.5)
    bad["x"][3, 2] = scene["res"][2] * scene["dx"] + 0.001
    bad["x"][4, 0] = -0.6 * scene["dx"]                          # stencil leaves the node grid below
    outs = []
    for via_append in (False, True):
        e = T.make_engine(scene, _cat(s1, bad)) if not via_append else T.make_engine(scene, s1)
        if via_append:
            _append(e, bad)
        n_live = e.num_particles()
        e.substep(1)
        outs.append((n_live, e.download()))
        e.close()
    assert outs[0][0] == outs[1][0]
    _assert_same(outs[0][1], outs[1][1])
    assert not np.isin(np.arange(len(s1["x"]), len(s1["x"]) + 5), outs[1][1]["id"]).any()


def _scattered(res, dx, n, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(8.0, np.asarray(res, np.float64) - 8.0, size=(n, 3))
    x = (X * dx).astype(np.float32)
    vol = np.full(n, np.float32(dx) ** 3 / 8, np.float32)
    return scenes.make_state(x, vol * 400, vol, scenes.MAT_JELLY)


@pytest.mark.parametrize("route", ["planes", "shapes", "dense"])
def test_delete_decisions_equal_the_mirrors_level_set_sample(route):
    res, dx = (36, 30, 41), float(np.float32(1.0 / 31))
    ls = mpm_mod.LevelSet(res, dx)
    if route == "planes":
        ls.add_plane((0.2, 1.0, -0.1), -0.55)
        ls.add_plane((-1.0, 0.1, 0.3), 0.8)
    else:
        ls.add_plane((0.2, 1.0, -0.1), -0.45)
        ls.add_sphere((0.6, 0.55, 0.7), 0.17)
        ls.add_cuboid((0.3, 0.3, 0.35), (0.95, 0.85, 1.2), inside_out=True)
    if route == "dense":
        ls.set_dense(scenes.shapes_sdf(res, ls.shapes_grid_units()))
    st = _scattered(res, dx, 6000, seed=len(route))
    scene = dict(res=res, dx=dx, dt=1e-4, gravity=(0.0, -10.0, 0.0), mat_kind=np.array([scenes.MAT_JELLY], np.int32),
                 mat_params=scenes.material_params(scenes.MAT_JELLY)[None])
    e = _bare_engine(scene)
    if route == "dense":
        e.set_sdf(ls.dense, 0.0)
    elif route == "shapes":
        e.set_levelset_shapes(ls.shapes_grid_units(), 0.0)
    else:
        e.set_planes(ls.planes_grid_units(), 0.0)
    e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    n_del = e.delete_inside_levelset()
    got = e.download()
    e.close()
    phi = ls.sample(st["x"].astype(np.float64) / dx)
    keep = np.zeros(len(phi), bool)
    keep[got["id"]] = True
    clear = np.abs(phi) >= 1e-5
    assert np.array_equal(keep[clear], ~(phi[clear] < 0))
    assert n_del == len(phi) - len(got["id"])
    assert 0.1 * len(phi) < n_del < 0.9 * len(phi)


def test_delete_keeps_survivors_bit_for_bit_and_later_substeps_follow_the_oracle():
    from oracle import pyoracle as O
    scene, st = T.perturbed_scene(scenes.MAT_SAND, res=32, cells=8, seed=5)
    e = T.make_engine(scene, st)
    e.substep(3)
    before = e.download()
    cut = np.array([[0.0, 1.0, 0.0, -13.0]], np.float32)         # the lower part of the block lies in the level set
    e.set_planes(cut, scene["friction"])
    n_del = e.delete_inside_levelset()
    after = e.download()
    keep = np.isin(before["id"], after["id"])
    assert n_del == len(before["id"]) - len(after["id"]) and 0 < n_del < len(before["id"])
    assert (before["x"][~keep][:, 1] / scene["dx"] < 13.0 + 1e-4).all() and (after["x"][:, 1] / scene["dx"] > 13.0 - 1e-4).all()
    _assert_same(after, {k: v[keep] for k, v in before.items()})
    scene2 = dict(scene, planes=cut, sdf=scenes.planes_sdf(32, cut))
    sv = _as_state(after)
    ref, _, _ = O.substep(scene2, sv, np.float64)
    e.substep(1)
    got = e.download()
    alive = ref["alive"].astype(bool)
    rows = np.searchsorted(after["id"], got["id"])
    assert np.array_equal(rows, np.nonzero(alive)[0])
    assert np.abs(got["x"] - ref["x"][rows]).max() <= T.TOL_X_ABS
    assert np.abs(got["v"] - ref["v"][rows]).max() <= T.TOL_V_REL * np.abs(ref["v"][alive]).max()
    assert np.abs(got["F"] - ref["F"][rows]).max() <= T.TOL_F_ABS
    assert T.ps_err(got["ps"], ref["ps"][rows]) <= T.TOL_PS_ABS
    # no level set: nothing is deleted
    e.set_sdf(None, 0.0)
    n = e.num_particles()
    assert e.delete_inside_levelset() == 0 and e.num_particles() == n
    e.close()


def test_rigid_colours_survive_an_append_and_a_delete():
    from tests.test_gpu_rigid import _engine, _scene
    scene, st, rigid = _scene()
    n = len(st["x"])
    e = _engine(scene, st, rigid)
    e.substep(2)
    c0 = e.get_particle_cdf(n)["states"]
    assert c0.any()
    extra = _take(st, slice(0, 16))
    extra["x"] = extra["x"] + np.float32(2 * scene["dx"])
    assert _append(e, extra) == n
    c1 = e.get_particle_cdf(n + 16)["states"]
    assert np.array_equal(c1[:n], c0) and not c1[n:].any()
    e.set_planes(np.array([[0.0, 1.0, 0.0, -float(np.median(st["x"][:, 1])) / scene["dx"]]], np.float32), 0.0)
    assert e.delete_inside_levelset() > 0
    assert np.array_equal(e.get_particle_cdf(n + 16)["states"], c1)
    e.substep(1)
    e.close()


def test_download_aos_after_an_append_reports_the_new_ids_and_touches_no_other_slot():
    # the reference's 320-byte slots, laid out as in test_gpu_parity.test_aos_round_trip
    scene, st = T.perturbed_scene(scenes.MAT_SAND, res=32, cells=4, seed=15)
    n = len(st["x"])
    L = capi.MpmbAosLayout()
    L.stride, L.off_v_and_m, L.off_pos, L.off_dg_e, L.off_apic_b, L.col_pitch = 320, 16, 32, 48, 96, 16
    L.off_vol, L.off_scalar = 164, 200
    slots = n + 7
    pool = np.zeros((slots, 320), np.uint8)
    indices = np.random.default_rng(1).permutation(slots)[:n].astype(np.uint32)
    f = pool.view(np.float32).reshape(slots, 80)
    for k, s in enumerate(indices):
        f[s, 4:7] = st["v"][k]; f[s, 7] = st["mass"][k]; f[s, 8:11] = st["x"][k]
        for c in range(3):
            f[s, 12 + 4 * c: 15 + 4 * c] = st["F"][k, 3 * c: 3 * c + 3]
        f[s, 41] = st["vol"][k]
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"])
    e.set_material(0, scenes.MAT_SAND, scene["mat_params"][0])
    e.upload_aos(pool, indices, L)
    e.substep(1)
    _append(e, _take(st, slice(0, 5)))
    resident = e.download()["id"]
    resident = resident[resident < n]
    pool0 = pool.copy()
    with pytest.raises(capi.MpmbError) as ex:
        e.download_aos(pool, indices.copy(), L)
    assert ex.value.code == -1                                   # MPMB_ERR_INVALID: ids past the index vector
    other = np.ones(slots, bool)
    other[indices[resident]] = False
    assert np.array_equal(pool[other], pool0[other])
    e.close()


def test_edits_are_refused_inside_a_substep_on_slab_ranks_and_past_the_id_range():
    scene, s1, s2 = _movers_scene(scenes.MAT_JELLY)
    e = T.make_engine(scene, s1)
    e.sort_particles_and_populate_grid()
    e.rasterize()
    for edit in (lambda: _append(e, s2), e.delete_inside_levelset):
        with pytest.raises(capi.MpmbError) as ex:
            edit()
        assert ex.value.code == -4                               # MPMB_ERR_STATE
    e.resample()
    assert _append(e, s2) == len(s1["x"])
    e.close()
    nt2 = (scene["res"][2] + 1 + 3) // 4 + 1
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], rank=0, world=2, tile_z0=0, tile_z1=nt2 // 2, migrate_capacity=4096)
    for edit in (lambda: _append(e, s2), e.delete_inside_levelset):
        with pytest.raises(capi.MpmbError) as ex:
            edit()
        assert ex.value.code == -4
    e.close()
    e = _bare_engine(scene)
    e.set_id_base(2 ** 28 - 10)
    e.upload(s1["x"][:4], s1["v"][:4], s1["mass"][:4], s1["vol"][:4])
    assert _append(e, _take(s2, slice(0, 6))) == 2 ** 28 - 6
    with pytest.raises(capi.MpmbError) as ex:
        _append(e, _take(s2, slice(0, 1)))
    assert ex.value.code == -3                                   # MPMB_ERR_CAPACITY
    e.close()


def test_mirror_edits_keep_ids_continue_the_span_and_match_the_download_upload_path(tmp_path):
    from scipy.spatial import cKDTree
    from taichi_mpm_b200 import bgeo

    def make(tag):
        m = mpm_mod.MPM(res=(32, 32, 32), base_delta_t=1e-4, frame_dt=5e-4, frame_directory=str(tmp_path / tag))
        ls = m.create_levelset()
        ls.add_plane((0, 1, 0), -0.25)
        ls.set_friction(0.4)
        m.set_levelset(ls)
        m.add_particles(type="sand", benchmark_block=((10, 10, 10), (14, 14, 14)), initial_velocity=(0.0, -0.5, 0.0))
        m.step(m.frame_dt)
        return m

    inlet = np.stack(np.meshgrid(*[np.arange(k) for k in (6, 2, 6)], indexing="ij"), -1).reshape(-1, 3)
    slab = ((inlet + 0.5) / 32 * 0.5 + np.array([0.55, 0.55, 0.4])).astype(np.float32)
    cut = mpm_mod.LevelSet((32, 32, 32), 1 / 32)
    cut.add_plane((0, 1, 0), -0.36)
    dev, old = make("dev"), make("old")
    for m in (dev, old):
        m.visualize()
    n0 = dev.num_particles()
    before = dev.get_particles()
    # append: on the device for `dev`; `old` holds a host copy, so it concatenates and uploads (the former path)
    for m in (dev, old):
        if m is old:
            m._pull_host()
        m.add_particles(type="water", positions=slab, initial_velocity=(0.0, -1.0, 0.0))
    p = dev.get_particles()
    assert np.array_equal(p["id"], np.arange(n0 + len(slab)))
    _assert_same({k: v[:n0] for k, v in p.items()}, before)
    for m in (dev, old):
        m.step(m.frame_dt)
        m.visualize()
    pos1, a1 = bgeo.read_bgeo(str(tmp_path / "dev" / "0001.bgeo"))
    pos2, a2 = bgeo.read_bgeo(str(tmp_path / "dev" / "0002.bgeo"))
    idx1, idx2 = dict((n, a) for n, _, a in a1)["index"].ravel(), dict((n, a) for n, _, a in a2)["index"].ravel()
    assert np.array_equal(idx1, np.arange(n0)) and np.array_equal(idx2, np.arange(n0 + len(slab)))     # visualize has the new ones
    # delete: survivors keep their ids and state on the device
    ids_before, mid = dev.get_particles()["id"], dev.get_particles()
    for m in (dev, old):
        m.set_levelset(cut)
        if m is old:
            m._pull_host()
        m.delete_particles_inside_level_set()
    p = dev.get_particles()
    assert 0 < len(p["id"]) < len(ids_before) and np.isin(p["id"], ids_before).all()
    keep = np.isin(mid["id"], p["id"])
    _assert_same(p, {k: v[keep] for k, v in mid.items()})
    span = n0 + len(slab)
    for m in (dev, old):
        if m is old:
            m._pull_host()
        m.add_particles(type="water", positions=slab + np.float32(0.05), initial_velocity=(0.0, -1.0, 0.0))
    p = dev.get_particles()
    assert np.array_equal(p["id"][-len(slab):], np.arange(span, span + len(slab)))   # after the span, not after the count
    for m in (dev, old):
        m.step(m.frame_dt)
        m.visualize()
    _, a3 = bgeo.read_bgeo(str(tmp_path / "dev" / "0003.bgeo"))
    assert np.array_equal(dict((n, a) for n, _, a in a3)["index"].ravel(), dev.get_particles()["id"])
    pd, po = dev.get_particles(), old.get_particles()
    assert len(pd["x"]) == len(po["x"])
    dist, j = cKDTree(po["x"]).query(pd["x"])
    assert len(np.unique(j)) == len(j) and dist.max() < 5e-5
    assert np.abs(pd["v"] - po["v"][j]).max() < 2e-2 * np.abs(po["v"]).max()
