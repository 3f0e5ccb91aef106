"""The affine matrix A = calculate_force() * (-4 dt / dx) + apic_b * 4 m that k_g2p (and every upload, append, seed and
material / step change) caches in the particle rows for the NEXT rasterize, checked against the fp64 oracle.  A is never
downloaded, but the next P2G's grid is a function of it: at any point between substeps the engine's next P2G must equal
the oracle's rasterize of the engine's current downloaded state, in which the oracle recomputes A from F, the plastic
scalar, apic_b and the mass itself.  The stress is a small part of a node's momentum, so the check isolates it: G_free is
the oracle's rasterize of the same state with F = I and the fresh plastic scalar (zero stress for every kind), and the
engine's error is measured against max |G_ref - G_free| instead of against the whole grid.  A probe with one particle
per tile also solves the next P2G for A particle by particle, at the branch edges of every material, and follows 20
substeps of those particles against 20 fp64 oracle substeps.  Runs on the SIMT emulator too
(tests/test_next_p2g_simt.py).  The rigid-coupled path (k_g2p_rigid) is checked the same way in
tests/test_gpu_rigid_parity.py; out of scope: the AsyncMPM pools (they rebuild A from the rows on every advance)."""
import numpy as np
import pytest

from taichi_mpm_b200 import capi, scenes
from tests import common as T

pytestmark = pytest.mark.gpu

# |G_eng - G_ref| on node momentum, relative to max |G_ref - G_free| (the stress part of the grid); a 1 % error of the
# stress (or of the apic term of the rows that carry it) is an error of order 1e-2 here.  Measured worst: 1.2e-4 (the
# arrivals scene, on an H100 and on the SIMT emulator alike), von Mises 9.7e-5, every other scene <= 3e-5; the table of
# DESIGN §2 lists them per test.
TOL_STRESS = 5e-4
# the stress part must be at least this fraction of max(|p|, m) over the grid, or the check above sees little
GUARD = 1e-4


def _take(st, sel):
    return {k: np.ascontiguousarray(v[sel]) for k, v in st.items()}


def _free_state(scene, S):
    """S with F = I and the fresh plastic scalar of every particle's kind: zero stress, the same mass, v and apic_b."""
    free = dict(S)
    free["F"] = np.tile(np.eye(3, dtype=np.float32).reshape(9), (len(S["x"]), 1))
    kinds = np.asarray(scene["mat_kind"])[np.asarray(S["group"])]
    free["ps"] = np.array([scenes.default_scalar(int(k)) for k in kinds], np.float32)
    return free


def _oracle_grids(scene, S):
    from oracle import pyoracle as O
    _, g_ref, _ = O.substep(scene, S, np.float64)
    _, g_free, _ = O.substep(scene, _free_state(scene, S), np.float64)
    return g_ref, g_free


def _grid_errors(g, g_ref, g_free, nodes=None):
    """Errors of the engine's P2G grid g against the oracle's (restricted to the boolean node mask `nodes`)."""
    stress = g_ref[..., :3] - g_free[..., :3]
    if nodes is not None:
        g, g_ref, stress = g[nodes], g_ref[nodes], stress[nodes]
    smax = np.abs(stress).max()
    gmax = max(np.abs(g_ref[..., :3]).max(), g_ref[..., 3].max())
    return dict(stress=float(np.abs(g[..., :3] - g_ref[..., :3]).max() / smax), visible=float(smax / gmax),
                grid=float(np.abs(g - g_ref).max() / gmax))


def _assert_grid(err, tol=TOL_STRESS, guard=GUARD):
    assert err["visible"] >= guard, err
    assert err["stress"] <= tol, err
    assert err["grid"] <= T.TOL_GRID_REL, err


def next_p2g(e, scene, label, tol=TOL_STRESS, guard=GUARD):
    """The engine's next P2G against the oracle's rasterize of its downloaded state; the engine then finishes the substep
    (resample), so that it can carry on.  Returns (errors, the state that was checked)."""
    S = e.download()
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g = e.download_grid(0).astype(np.float64)
    e.resample()
    err = _grid_errors(g, *_oracle_grids(scene, S))
    print(label, {k: "%.3g" % v for k, v in err.items()})
    _assert_grid(err, tol, guard)
    return err, S


# ---------------------------------------------------------------------------------------------------- k_g2p, every kind
KINDS = [("linear", scenes.MAT_LINEAR), ("jelly", scenes.MAT_JELLY), ("snow", scenes.MAT_SNOW), ("water", scenes.MAT_WATER),
         ("sand", scenes.MAT_SAND), ("elastic", scenes.MAT_ELASTIC), ("von_mises", scenes.MAT_VON_MISES), ("visco", scenes.MAT_VISCO)]


@pytest.mark.parametrize("no_graph", [False, True], ids=["graph", "no_graph"])
@pytest.mark.parametrize("nsub", [0, 1, 2, 7])
@pytest.mark.parametrize("name,kind", KINDS)
def test_next_p2g_after_substeps(name, kind, nsub, no_graph):
    # nsub = 0: the A of the upload (pack_one); 1: of one k_g2p that stores apic_b; 2 and 7: the middle substeps of one
    # substep(n) call skip the apic_b streams (STORE_B = false), the last one stores them.  Slow particles: the stress is
    # then a larger part of the node momentum.
    scene, st = T.perturbed_scene(kind, res=32, cells=6, seed=3, vel=0.05, **T.KIND_KW.get(kind, {}))
    e = T.make_engine(scene, st, no_graph=no_graph)
    if nsub:
        e.substep(nsub)
    next_p2g(e, scene, "%s nsub=%d no_graph=%d" % (name, nsub, no_graph))
    e.close()


@pytest.mark.parametrize("name,kind", KINDS)
def test_one_call_of_n_substeps_equals_n_calls_of_one(name, kind):
    # the A of a middle substep (STORE_B = false, apic_b only in registers) is consumed inside the same substep(n) call and
    # never seen between calls: n calls of substep(1), where every G2P stores apic_b, must end on the same bits
    scene, st = T.perturbed_scene(kind, res=32, cells=6, seed=3, vel=0.05, **T.KIND_KW.get(kind, {}))
    outs = []
    for calls, no_graph in (((7,), False), ((7,), True), ((1,) * 7, False), ((3, 1, 3), True)):
        e = T.make_engine(scene, st, no_graph=no_graph)
        for n in calls:
            e.substep(n)
        outs.append(e.download())
        e.close()
    for o in outs[1:]:
        for k in ("id", "x", "v", "F", "b", "ps"):
            assert np.array_equal(o[k], outs[0][k]), k


# ---------------------------------------------------------------------------------------------------- arrivals
def test_next_p2g_after_substeps_with_arrivals():
    # rows that changed tile in the last G2P are the next P2G's arrival rows: stored with a negated mass, their A must
    # still carry +|m| in the apic term.  The scene of test_gpu_geometry's movers test, with strained sand (so that the
    # stress is visible next to its fast particles).
    from tests.test_gpu_geometry import _movers_scene
    scene, st = _movers_scene()
    rng = np.random.default_rng(19)
    st["F"] = (st["F"] + rng.normal(size=st["F"].shape) * 0.01).astype(np.float32)
    for no_graph in (False, True):
        e = T.make_engine(scene, st, no_graph=no_graph)
        e.substep(11)
        e.substep(1)
        arrivals = e.get_ordering_stats()["movers"]
        assert arrivals > 20, arrivals
        next_p2g(e, scene, "arrivals no_graph=%d (%d arrival rows)" % (no_graph, arrivals))
        e.close()


# ---------------------------------------------------------------------------------------------------- several groups
def mixed_state(res, lo, hi, kinds, seed, strain=0.02, vel=0.05, groups=None):
    """A jittered lattice block whose particles belong to groups 0 .. len(kinds) - 1 (random, interleaved, or `groups`),
    each perturbed as perturbed_scene perturbs a block of its group's kind."""
    x, mass, vol = scenes.lattice_block(res, lo, hi, jitter=0.2, seed=seed + 1)
    n = len(x)
    rng = np.random.default_rng(seed)
    g = rng.integers(0, len(kinds), n).astype(np.int32) if groups is None else np.asarray(groups, np.int32)
    st = scenes.make_state(x, mass, vol, scenes.MAT_JELLY)
    st["group"] = g
    st["ps"] = np.zeros(n, np.float32)
    for k, kind in enumerate(kinds):
        sel = np.nonzero(g == k)[0]
        sub = _take(st, sel)
        T.perturb_state(sub, kind, 1.0 / res, seed + 7 * k, strain, vel)
        for key in ("v", "b", "F", "ps"):
            st[key][sel] = sub[key]
    return st


def mixed_scene(res, kinds, params, dt=5e-5):
    planes = np.array([[0.0, 1.0, 0.0, -8.6]], np.float32)
    return dict(res=(res, res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0, 0.0), particle_gravity=1,
                mat_kind=np.array(kinds, np.int32), mat_params=np.array(params, np.float32), planes=planes, friction=0.4,
                sdf=scenes.planes_sdf(res, planes))


def test_next_p2g_after_set_material_and_set_delta_t():
    # k_refresh_affine rebuilds A of one group (set_material) or of every group (set_delta_t) from the stored F, scalar
    # and apic_b; groups other than 0 must get their own material and the new step
    kinds = [scenes.MAT_JELLY, scenes.MAT_SNOW, scenes.MAT_SAND, scenes.MAT_VISCO]
    params = [scenes.material_params(k) for k in kinds]
    params[3] = scenes.material_params(scenes.MAT_VISCO, kappa=0.3)
    scene = mixed_scene(32, kinds, params)
    st = mixed_state(32, (12, 9, 12), (20, 17, 20), kinds, seed=41, strain=0.01)
    e = T.make_engine(scene, st)
    e.substep(3)
    for g, kind, kw in ((1, scenes.MAT_SNOW, dict(youngs_modulus=3e5, hardening=5.0)), (2, scenes.MAT_SAND, dict(friction_angle=40.0, cohesion=1e-3)),
                        (3, scenes.MAT_VISCO, dict(youngs_modulus=8e4, kappa=0.3))):
        scene["mat_params"][g] = scenes.material_params(kind, **kw)
        e.set_material(g, kind, scene["mat_params"][g])
    next_p2g(e, scene, "set_material groups 1-3")
    e.substep(2)
    for dt in (3e-5, 7e-5):
        scene["dt"] = dt
        e.set_delta_t(dt)
        next_p2g(e, scene, "set_delta_t %g" % dt)
        e.substep(2)
    e.close()


# ---------------------------------------------------------------------------------------------------- all 16 groups
# groups 8 .. 15: the kinds of groups 0 .. 7 with parameters other than the defaults
GROUP_KW = {8: dict(E=2e5, nu=0.25), 9: dict(E=5e4, nu=0.2), 10: dict(hardening=5.0), 11: dict(gamma=3.0),
            12: dict(friction_angle=40.0, cohesion=1e-3), 13: dict(E=1e4), 14: dict(yield_stress=0.5), 15: dict(kappa=0.3)}
# sand's series path: bounds of |F F^T - I|_F^2 where sym_log1p_series changes its term count, and the 0.15^2 above which
# the lane takes the eigen path (mpmb_math.cuh)
SAND_SERIES_EDGES = [4.0e-7, 6.2e-5, 7.8e-4, 3.5e-3, 9.2e-3, 0.0225]


def _sixteen_groups(seed=61):
    kinds = [g % 8 for g in range(16)]
    params = [scenes.material_params(k, **GROUP_KW.get(g, {})) for g, k in enumerate(kinds)]
    scene = mixed_scene(32, kinds, params, dt=2e-5)
    st = mixed_state(32, (10, 9, 10), (20, 15, 20), kinds, seed=seed, strain=0.006)
    # sand strains spread over the term-count bins and both sides of the series / eigen switch, interleaved with the rest,
    # so that warp_max_active and __any_sync run over lanes that want different branches.  Which term count a warp then
    # takes is its lanes' maximum on the trial F: the histogram below shows the mix, not that every count runs; one
    # particle per warp does that (test_isolated_particles_affine_per_particle_and_trajectories).
    rng = np.random.default_rng(seed + 1)
    sand = np.nonzero(np.asarray(kinds)[st["group"]] == scenes.MAT_SAND)[0]
    s = 10.0 ** rng.uniform(-4.5, -1.0, len(sand))
    st["F"][sand] = (np.eye(3).reshape(9) + rng.normal(size=(len(sand), 9)) * s[:, None]).astype(np.float32)
    F = st["F"][sand].reshape(-1, 3, 3).transpose(0, 2, 1).astype(np.float64)
    nE2 = ((F @ F.transpose(0, 2, 1) - np.eye(3)) ** 2).sum((1, 2))
    counts = np.histogram(nE2, [0.0] + SAND_SERIES_EDGES + [np.inf])[0]
    assert (counts >= 5).all(), counts
    return scene, st


def test_sixteen_groups_interleaved():
    from tests.test_gpu_parity import _assert_parity
    scene, st = _sixteen_groups()
    assert len(np.unique(st["group"])) == 16
    # every warp of k_g2p sees several kinds
    e = T.make_engine(scene, st)
    err, _, _ = T.compare_substep(e, scene, st)
    print("16 groups, first substep", {k: (float(v) if not isinstance(v, bool) else v) for k, v in err.items()})
    _assert_parity(err)
    e.substep(4)
    next_p2g(e, scene, "16 groups, 5 substeps")
    e.substep(3)
    next_p2g(e, scene, "16 groups, 9 substeps")
    e.close()


def test_sixteen_groups_with_nan_tags():
    # at id_base = 2^28 - n - 8 the tag (group << 28 | id) of every particle of groups 7 and 15 is a NaN bit pattern as
    # a float: the run must not care, and ids and groups must come back exactly
    scene, st = _sixteen_groups(seed=67)
    n = len(st["x"])
    base = 2 ** 28 - n - 8
    tags = (st["group"].astype(np.uint32) << np.uint32(28)) | (np.uint32(base) + np.arange(n, dtype=np.uint32))
    assert np.isnan(tags.view(np.float32)[np.isin(st["group"], (7, 15))]).all()
    outs = []
    for b in (0, base):
        e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"])
        for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
            e.set_material(g, int(k), p)
        e.set_planes(scene["planes"], scene["friction"])
        e.set_id_base(b)
        e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
        e.substep(6)
        d = e.download()
        nb, recs = e.download_bgeo_points(n)
        pool, indices, L = _aos_pool(st, 3)
        idx = indices.copy()
        n_aos = e.download_aos(pool, idx, L)
        if b:
            next_p2g(e, scene, "16 groups, NaN tags")
        e.close()
        outs.append((d, nb, recs, pool, indices, idx, n_aos))
    (d0, _, _, _, _, _, _), (d1, nb, recs, pool, indices, idx, n_aos) = outs
    assert len(d1["id"]) == len(d0["id"]) > n // 2
    assert np.array_equal(d1["id"] - np.uint32(base), d0["id"]) and np.array_equal(d1["group"], d0["group"])
    assert np.array_equal(d0["group"], st["group"][d0["id"]])
    for k in ("x", "v", "F", "b", "ps", "mass", "vol"):
        assert np.array_equal(d1[k].view(np.uint32), d0[k].view(np.uint32)), k
    # the frame dump's point records carry the absolute id (word 5, big-endian), in id order
    assert nb == len(d1["id"])
    w = recs.view(">u4").reshape(nb, 12)
    assert np.array_equal(w[:, 5], d1["id"]) and np.array_equal(w[:, :3].view(">f4").astype(np.float32), d1["x"])
    # the reference's slots: particle k of the survivors (id order) back in the slot of its id
    assert n_aos == len(d1["id"])
    assert np.array_equal(idx[:n_aos], indices[d0["id"]])
    f = pool.view(np.float32).reshape(len(pool), 80)
    assert np.array_equal(f[idx[:n_aos], 8:11], d1["x"]) and np.array_equal(f[idx[:n_aos], 4:7], d1["v"])


# ---------------------------------------------------------------------------------------------------- z slabs
def _slab_next_p2g(S, scene, label):
    """next_p2g for the engines of a z-slab run in one process (peer exchange): every rank's owned node layers (z in
    [4 z0, 4 z1)) after the halo exchange against the oracle's rasterize of the union of the ranks' states."""
    parts = [e.download() for e in S.eng]
    U = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    for e in S.eng:
        e.sort_particles_and_populate_grid()
        e.rasterize()
    for f_e in (lambda e, f: e.halo_send(f), lambda e, f: e.halo_recv(f)):
        for r, e in enumerate(S.eng):
            for f in S.faces[r]:
                f_e(e, f)
    grids = [e.download_grid(0).astype(np.float64) for e in S.eng]
    for e in S.eng:
        e.resample()
    for f_e in (lambda e, f: e.migrate_send(f), lambda e, f: e.migrate_recv(f)):
        for r, e in enumerate(S.eng):
            for f in S.faces[r]:
                f_e(e, f)
    g_ref, g_free = _oracle_grids(scene, U)
    z = np.arange(g_ref.shape[2])
    for r, (z0, z1) in enumerate(S.cuts):
        owned = np.zeros(g_ref.shape[:3], bool)
        owned[:, :, (z >= 4 * z0) & (z < 4 * z1)] = True
        owned &= g_ref[..., 3] > 0
        err = _grid_errors(grids[r], g_ref, g_free, owned)
        print(label, "rank %d of %d (%d particles)" % (r, S.world, len(parts[r]["id"])), {k: "%.3g" % v for k, v in err.items()})
        _assert_grid(err)


@pytest.mark.parametrize("world", [2, 3])
def test_next_p2g_on_z_slabs_after_migration_and_recut(world):
    # rows that crossed a slab cut (migration) and rows moved to a new owner by a re-cut carry their A with them
    from tests.test_gpu_slab import _scene
    from tests.test_gpu_slab_edit import _Slabs
    from tests.test_gpu_slab_recut import _recut
    scene, st = _scene()
    rng = np.random.default_rng(71)
    st["F"] = (st["F"] + rng.normal(size=st["F"].shape) * 0.01).astype(np.float32)
    S = _Slabs(scene, st, world, peer=True)
    S.step(6)
    _slab_next_p2g(S, scene, "slabs after migration")
    flat = [S.cuts[0][0]] + [z1 for _, z1 in S.cuts]
    flat[1:-1] = [c + 1 for c in flat[1:-1]]
    _, _, moved = _recut(S, [(a, b) for a, b in zip(flat[:-1], flat[1:])])
    assert moved > 0
    _slab_next_p2g(S, scene, "slabs after recut")
    S.close()


# ---------------------------------------------------------------------------------------------------- isolated particles
# One particle per 4^3-cell tile, its base node at 4 k + 1 on every axis: no node is shared, so the 27 nodes of a
# particle give p_n = w_n (m v + A d_n), m_n = w_n m (d_n = particle - node, grid units) and A can be solved for per
# particle.  Alone in its tile, a particle is also alone in its warp: warp_max_active and __any_sync take its own branch.
PROBE_RES, PROBE_SLOTS = 64, 12
PROBE_DT = 2e-5
PROBE_KINDS = [scenes.MAT_SAND, scenes.MAT_SNOW, scenes.MAT_WATER, scenes.MAT_VON_MISES, scenes.MAT_VISCO, scenes.MAT_JELLY,
               scenes.MAT_LINEAR, scenes.MAT_ELASTIC]
PROBE_KW = {scenes.MAT_SAND: dict(cohesion=1e-3), scenes.MAT_WATER: dict(k=10.0, gamma=3.0), scenes.MAT_VISCO: dict(kappa=0.3)}
SAND_EDGES = [0.0] + SAND_SERIES_EDGES[:-1] + [0.0225, 0.1, np.inf]   # the term-count bins, the 0.15 switch, the eigen path


def _math(a9):
    """column-major 9-vectors -> 3x3 matrices (math layout)"""
    return np.asarray(a9, np.float64).reshape(-1, 3, 3).transpose(0, 2, 1)


def _sand_case(Ft, prm, ps):
    """SandParticle::project's case (0 expansion, 1 inside the cone, 2 projected) and |Ft Ft^T - I|_F^2, in fp64."""
    s = np.linalg.svd(Ft, compute_uv=False)
    eps = np.log(np.maximum(np.abs(s), 1e-4)) - prm[3]
    tr = eps.sum(1) + ps
    hat = eps - tr[:, None] / 3
    dg = np.linalg.norm(hat, axis=1) + (3 * prm[1] + 2 * prm[0]) / (2 * prm[0]) * tr * prm[2]
    case = np.where(tr >= 0, 0, np.where(dg <= 0, 1, 2))
    nE2 = ((Ft @ Ft.transpose(0, 2, 1) - np.eye(3)) ** 2).sum((1, 2))
    return case, nE2


def _probe_state(seed=81):
    rng = np.random.default_rng(seed)
    dx = 1.0 / PROBE_RES
    ks = np.stack(np.meshgrid(*[np.arange(2, 2 + PROBE_SLOTS)] * 3, indexing="ij"), -1).reshape(-1, 3)
    ks = ks[rng.permutation(len(ks))]
    params = [scenes.material_params(k, **PROBE_KW.get(k, {})) for k in PROBE_KINDS]
    Fs, pss, groups = [], [], []
    # sand: every bin of SAND_EDGES in every case of the return map (chosen on the uploaded F; checked on the trial F)
    pool = []
    for _ in range(40):
        s = 10.0 ** rng.uniform(-4.2, -0.6, 1000)
        D = rng.normal(size=(1000, 3, 3))
        D = 0.5 * (D + D.transpose(0, 2, 1))
        D -= np.trace(D, axis1=1, axis2=2)[:, None, None] / 3 * np.eye(3)
        D /= np.linalg.norm(D, axis=(1, 2))[:, None, None]
        u = rng.uniform(-1.0, 1.0, 1000)
        F = np.eye(3) + s[:, None, None] * (D * np.sqrt(1 - u ** 2)[:, None, None] + u[:, None, None] * np.eye(3) / np.sqrt(3))
        # logJp: 0, of the order of the strain, or near 3 * cohesion (where tiny strains reach the apex and the cone)
        r = rng.random(1000)
        ps = np.where(r < 0.3, rng.uniform(0, 3, 1000) * s, np.where(r < 0.6, 3 * params[0][3] + rng.uniform(-2, 2, 1000) * s, 0.0))
        case, nE2 = _sand_case(F, params[0], ps)
        pool.append((F, ps, case, np.digitize(nE2, SAND_EDGES) - 1))
    F, ps, case, b = (np.concatenate(a) for a in zip(*pool))
    for bn in range(len(SAND_EDGES) - 1):
        for c in range(3):
            idx = np.nonzero((b == bn) & (case == c))[0][:8]
            Fs.append(F[idx]); pss.append(ps[idx]); groups.append(np.zeros(len(idx), np.int32))
    # snow: singular values on both sides of [1 - theta_c, 1 + theta_s]; Jp at both clamps
    n = 120
    R, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    sig = rng.uniform(0.95, 1.03, (n, 3))
    F = R @ (sig[:, :, None] * R.transpose(0, 2, 1))
    jp = np.where(sig.min(1) < 0.975, 0.6, np.where(sig.max(1) > 1.0075, 20.0, 1.0))
    jp = np.where(rng.random(n) < 0.5, jp, rng.uniform(0.8, 1.5, n))
    Fs.append(F); pss.append(jp); groups.append(np.full(n, 1, np.int32))
    # water at the j = 0.1 floor (compressed: apic_b below has a positive trace) and away from it
    n = 80
    Fs.append(np.tile(np.eye(3), (n, 1, 1))); pss.append(np.where(np.arange(n) % 2 == 0, 0.1, rng.uniform(0.9, 1.1, n)))
    groups.append(np.full(n, 2, np.int32))
    # von Mises on both sides of the yield surface; visco, jelly, linear, elastic at moderate strain
    for g, strain, n in ((3, 0.006, 120), (4, 0.05, 80), (5, 0.02, 60), (6, 0.02, 60), (7, 0.05, 60)):
        Fs.append(np.eye(3) + rng.normal(size=(n, 3, 3)) * strain)
        pss.append(1000.0 * (0.2 + 1.6 * rng.random(n)) if g == 4 else np.zeros(n))
        groups.append(np.full(n, g, np.int32))
    F = np.concatenate(Fs)
    n = len(F)
    assert n <= len(ks), n
    base = 4 * ks[:n] + 1
    X = base + rng.uniform(0.6, 1.4, (n, 3))
    x = (X * dx).astype(np.float32)
    vol = np.full(n, dx ** 3 / 8, np.float32)
    st = scenes.make_state(x, (vol * 400).astype(np.float32), vol, scenes.MAT_JELLY)
    st["F"] = np.ascontiguousarray(F.transpose(0, 2, 1).reshape(n, 9), np.float32)
    st["ps"] = np.concatenate(pss).astype(np.float32)
    st["group"] = np.concatenate(groups)
    st["v"] = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32)
    b = rng.normal(size=(n, 3, 3)) * 1e-3
    b[st["group"] == 2] += 0.1 * np.eye(3)    # compression that outweighs the pressure of j = 0.1
    st["b"] = np.ascontiguousarray(b.transpose(0, 2, 1).reshape(n, 9), np.float32)
    scene = dict(res=(PROBE_RES,) * 3, dx=dx, dt=PROBE_DT, gravity=(0.0, -10.0, 0.0), particle_gravity=1,
                 mat_kind=np.array(PROBE_KINDS, np.int32), mat_params=np.array(params, np.float32), planes=None, friction=0.0, sdf=None)
    return scene, st


def _recover_affine(g, S, dx):
    """A of every particle of S (id order) from its 27 nodes of the P2G grid g: least squares of p_n = m_n (v + A d_n / m)."""
    X = S["x"].astype(np.float32) * (np.float32(1.0) / np.float32(dx))
    base = (X - np.float32(0.5)).astype(np.int32)
    rel = X.astype(np.float64) - base
    off = np.stack(np.meshgrid(*[np.arange(3)] * 3, indexing="ij"), -1).reshape(27, 3)
    nodes = base[:, None, :] + off[None]
    gn = g[nodes[..., 0], nodes[..., 1], nodes[..., 2]]                      # (n, 27, 4)
    d = rel[:, None, :] - off[None]
    M = gn[..., 3:4] * np.concatenate([np.ones((len(X), 27, 1)), d], 2)      # (n, 27, 4)
    C = np.stack([np.linalg.lstsq(M[i], gn[i, :, :3], rcond=None)[0] for i in range(len(X))])
    return S["mass"].astype(np.float64)[:, None, None] * C[:, 1:, :].transpose(0, 2, 1)


def _probe(e, scene, label):
    """Downloaded state, A recovered from the next P2G, A the oracle computes from that state (fp64)."""
    from oracle import pyoracle as O
    S = e.download()
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g = e.download_grid(0).astype(np.float64)
    e.resample()
    A = _recover_affine(g, S, scene["dx"])
    S_ = -4.0 / float(np.float32(scene["dx"])) * scene["dt"]
    Fm, bm = _math(S["F"]), _math(S["b"])
    stress = np.stack([O.calculate_force(int(scene["mat_kind"][gr]), scene["mat_params"][gr], Fm[i], float(S["ps"][i]), float(S["vol"][i])) * S_
                       for i, gr in enumerate(S["group"])])
    ref = stress + 4.0 * S["mass"].astype(np.float64)[:, None, None] * bm
    worst = {}
    for gr, k in enumerate(PROBE_KINDS):
        sel = S["group"] == gr
        # per particle: relative to its own stress term, with a floor of 1e-2 of the kind's largest one
        scale = np.abs(stress[sel]).max((1, 2)) + 1e-2 * np.abs(stress[sel]).max()
        worst[KINDS[k][0]] = float((np.abs(A[sel] - ref[sel]).max((1, 2)) / scale).max())
    print(label, {k: "%.3g" % v for k, v in worst.items()})
    return worst, S


def test_isolated_particles_affine_per_particle_and_trajectories():
    from oracle import pyoracle as O
    scene, st = _probe_state()
    n = len(st["x"])
    # the branches, with numpy on the trial state of the first substep (Ft = cdg F, cdg = I + S b' from the oracle's b')
    r1, _, _ = O.substep(scene, st, np.float64)
    assert r1["alive"].all()
    S_ = -4.0 / float(np.float32(scene["dx"])) * scene["dt"]
    Ft = (np.eye(3) + S_ * _math(r1["b"])) @ _math(st["F"])
    g = st["group"]
    sand = g == 0
    case, nE2 = _sand_case(Ft[sand], scene["mat_params"][0].astype(np.float64), st["ps"][sand].astype(np.float64))
    bins = np.digitize(nE2, SAND_EDGES) - 1
    hit = {(int(bn), int(c)) for bn, c in zip(bins, case)}
    missing = [(bn, c) for bn in range(len(SAND_EDGES) - 1) for c in range(3) if (bn, c) not in hit]
    assert not missing, missing
    snow = g == 1
    sg = np.linalg.svd(Ft[snow], compute_uv=False)
    assert (sg.min(1) < 0.975).any() and (sg.max(1) > 1.0075).any()
    min_jp, max_jp = (float(scene["mat_params"][1][k]) for k in (5, 6))
    assert (r1["ps"][snow] == min_jp).any() and (r1["ps"][snow] == max_jp).any()
    water = g == 2
    assert (r1["ps"][water] == 0.1).any() and (r1["ps"][water] > 0.5).any()
    # visco: the halving loop of approximate_exponent runs only when det(I + s + s^2 / 2) <= 0 (s = cdg - I), and every
    # eigenvalue factor 1 + l + l^2 / 2 of that matrix is positive for real l and |.|^2 >= 0 for a complex pair: the loop
    # is reachable only through rounding at l = -1 +- i, so no particle is placed there; its visco particles flow (tau moves)
    visco = g == 4
    assert (np.abs(r1["ps"][visco] - st["ps"][visco]) > 1e-3).any()
    vm = g == 3
    eps = np.log(np.linalg.svd(Ft[vm], compute_uv=False))
    n2 = ((eps - eps.mean(1, keepdims=True)) ** 2).sum(1)
    yielding = n2 > scene["mat_params"][3][2] / (2 * scene["mat_params"][3][0])
    assert 0.1 < yielding.mean() < 0.9, yielding.mean()
    # A after one substep, and after a substep(20) call, against the trajectory of 20 fp64 oracle substeps
    e = T.make_engine(scene, st)
    e.substep(1)
    w1, _ = _probe(e, scene, "isolated, 1 substep")
    e.close()
    e = T.make_engine(scene, st)
    e.substep(20)
    d = e.download()
    w20, _ = _probe(e, scene, "isolated, 20 substeps")
    e.close()
    ref = dict(st)
    for _ in range(20):
        ref, _, _ = O.substep(scene, ref, np.float64, want_grids=False)
    assert ref["alive"].all() and np.array_equal(d["id"], np.arange(n))
    err = dict(x=np.abs(d["x"] - ref["x"]).max(), v=np.abs(d["v"] - ref["v"]).max() / np.abs(ref["v"]).max(),
               b=np.abs(d["b"] - ref["b"]).max() / np.abs(ref["b"]).max(), F=np.abs(d["F"] - ref["F"]).max(), ps=T.ps_err(d["ps"], ref["ps"]))
    ps_kind = {KINDS[k][0]: T.ps_err(d["ps"][g == gr], ref["ps"][g == gr]) for gr, k in enumerate(PROBE_KINDS)}
    print("isolated, 20-substep trajectories", {k: "%.3g" % v for k, v in err.items()}, "ps by kind", {k: "%.3g" % v for k, v in ps_kind.items()})
    for w in (w1, w20):
        assert max(w.values()) <= PROBE_TOL_A, w
    # single-substep tolerances (tests/common.py), except the plastic scalar, which sums 20 steps of rounding
    assert err["x"] <= T.TOL_X_ABS and err["v"] <= T.TOL_V_REL and err["b"] <= T.TOL_V_REL, err
    assert err["F"] <= T.TOL_F_ABS and err["ps"] <= PROBE_TOL_PS, err


# recovered A against the oracle's, per particle, relative to its own stress term plus 1e-2 of its kind's largest
PROBE_TOL_A = 1e-3
PROBE_TOL_PS = 5e-4


# ---------------------------------------------------------------------------------------------------- uploads and edits
def test_next_p2g_after_append():
    # the appended rows' A comes from pack_one (several groups, none of them group 0's material); the resident rows' A
    # from the last k_g2p
    kinds = [scenes.MAT_JELLY, scenes.MAT_SNOW, scenes.MAT_SAND]
    scene = mixed_scene(32, kinds, [scenes.material_params(k) for k in kinds])
    st = mixed_state(32, (10, 9, 10), (22, 15, 22), kinds, seed=43, strain=0.01)
    first = st["x"][:, 0] < 0.5
    s1, s2 = _take(st, first), _take(st, ~first)
    e = T.make_engine(scene, s1)
    e.substep(3)
    assert e.append(s2["x"], s2["v"], s2["mass"], s2["vol"], s2["F"], s2["b"], s2["ps"], s2["group"]) == len(s1["x"])
    next_p2g(e, scene, "append")
    e.substep(2)
    next_p2g(e, scene, "append + 2 substeps")
    e.close()


def _aos_pool(st, seed):
    L = capi.MpmbAosLayout()
    L.stride, L.off_v_and_m, L.off_pos, L.off_dg_e, L.off_apic_b, L.col_pitch = 320, 16, 32, 48, 96, 16
    L.off_vol, L.off_scalar = 164, 200
    n = len(st["x"])
    slots = n + 7
    pool = np.zeros((slots, 320), np.uint8)
    indices = np.random.default_rng(seed).permutation(slots)[:n].astype(np.uint32)
    f = pool.view(np.float32).reshape(slots, 80)
    f[indices, 4:7] = st["v"]; f[indices, 7] = st["mass"]; f[indices, 8:11] = st["x"]
    for c in range(3):
        f[indices, 12 + 4 * c: 15 + 4 * c] = st["F"][:, 3 * c: 3 * c + 3]
        f[indices, 24 + 4 * c: 27 + 4 * c] = st["b"][:, 3 * c: 3 * c + 3]
    f[indices, 41] = st["vol"]
    f[indices, 50] = st["ps"]
    return pool, indices, L


def test_next_p2g_after_upload_aos():
    kinds = [scenes.MAT_JELLY, scenes.MAT_SAND, scenes.MAT_SNOW]
    scene = mixed_scene(32, kinds, [scenes.material_params(k) for k in kinds])
    st = mixed_state(32, (12, 9, 12), (20, 15, 20), kinds, seed=45, strain=0.01)
    pool, indices, L = _aos_pool(st, 2)
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"])
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    e.set_planes(scene["planes"], scene["friction"])
    e.upload_aos(pool, indices, L, group=st["group"])
    next_p2g(e, scene, "upload_aos")
    e.close()


@pytest.mark.parametrize("group", [1, 3])
def test_next_p2g_after_seed_lattice(group):
    # seeded rows start at F = I, apic_b = 0 and the fresh scalar of their group's kind (snow: Jp = 1; visco: 0): zero
    # stress, so their A is 0.  Strained particles appended beside the block (other groups) give the stress the check sees.
    kinds = [scenes.MAT_JELLY, scenes.MAT_SNOW, scenes.MAT_SAND, scenes.MAT_VISCO]
    scene = mixed_scene(32, kinds, [scenes.material_params(k) for k in kinds])
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"])
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    e.set_planes(scene["planes"], scene["friction"])
    vol = np.float32(scene["dx"]) ** 3 / 8
    n_seeded = e.seed_lattice((10, 9, 10), (16, 14, 16), vol, vol * 400, jitter=0.2, seed=5, group=group, v0=(0.3, -0.2, 0.1))
    assert n_seeded > 1000
    st = mixed_state(32, (16, 9, 10), (22, 14, 16), kinds[:3:2], seed=47, strain=0.01)   # groups 0 and 1 ...
    st["group"] = np.where(st["group"] == 1, 2, 0).astype(np.int32)                        # ... as jelly and sand
    e.append(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    next_p2g(e, scene, "seed_lattice group %d" % group)
    e.substep(2)
    next_p2g(e, scene, "seed_lattice group %d + 2 substeps" % group)
    e.close()
