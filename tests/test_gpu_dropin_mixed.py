"""The drop-in for pools that mix particle types (INTEGRATION.md §2, MpmbAosLayout.off_scalar_by_kind): every type keeps its
plastic scalar at its own offset of the slot (snow Jp, water j, sand logJp, visco visco_tau), and the offset of a row follows
the material kind of its group.

  * byte round trip: a pool of all eight types plus a second sand and snow group, every slot filled with noise around the
    fields, comes back from mpmb_upload_aos -> mpmb_download_aos byte for byte, indices too, also after mpmb_set_material has
    changed a group's kind in between (the download follows the upload's snapshot); the uploaded scalars are the slot's or
    the kind's default;
  * refusal: a per-kind layout with off_scalar != -1 or an entry that is not a 4-aligned offset in (0, stride - 4] is
    refused by both calls and changes nothing;
  * the reference's own MPM<3> object steps a mixed pool by itself and through the C-ABI (oracle/transfer_mixed_ref.cpp),
    and its AsyncMPM<3> scheduler is routed through one engine on sand + elastic and on snow + water;
  * 1 M particles of four types in four blocks: the byte round trip, and one substep equal bit for bit to the substep after
    mpmb_upload_particles of the same particles.

Reads only oracle/_ref (the reference's objects built there); tests/test_dropin_mixed.py runs the same on the SIMT emulator."""
import numpy as np
import pytest

from oracle import pyoracle_mixed as M
from taichi_mpm_b200 import capi, scenes

# the slot layout comes from offsetof() on the reference's classes (oracle/_ref)
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not M.ref_available(), reason="reference build (oracle/_ref) not available")]

RES, DX, DT = 32, 1.0 / 32, 2e-5
STRIDE = 320
# (kind, material keywords) per group: group numbers differ from the kinds, and sand and snow come twice with other parameters
GROUPS = [(scenes.MAT_SAND, {}), (scenes.MAT_SNOW, {}), (scenes.MAT_VISCO, {}), (scenes.MAT_WATER, {}), (scenes.MAT_LINEAR, {}),
          (scenes.MAT_ELASTIC, {}), (scenes.MAT_JELLY, {}), (scenes.MAT_VON_MISES, {}), (scenes.MAT_SAND, dict(cohesion=0.05)),
          (scenes.MAT_SNOW, dict(hardening=5.0))]


def reference_layout():
    """The reference's slot layout, offsetof() on its own classes (oracle/_ref), with the per-kind scalar offsets."""
    from oracle import pyoracle_mixed as M
    lay = M.aos_layout()
    L = capi.MpmbAosLayout()
    L.stride, L.off_pos, L.off_v_and_m, L.off_dg_e, L.off_apic_b, L.col_pitch, L.off_vol = (int(v) for v in lay[:7])
    off = M.aos_scalar_offsets()
    L.set_scalar_offsets(dict(zip(capi.MpmbAosLayout.SCALAR_KINDS, (int(o) for o in off))))
    return L


def mixed_scene(groups=GROUPS, res=RES, cells=3, seed=3, dt=DT):
    """One block of `cells`^3 cells per group, side by side along x and z (they collide), each perturbed as its type; every
    plastic scalar is away from its default."""
    from tests import common as T
    parts, kinds, prms = [], [], []
    for g, (kind, kw) in enumerate(groups):
        lo = np.array([8 + cells * (g % 5), 9, 11 + cells * (g // 5)])
        x, mass, vol = scenes.lattice_block(res, lo, lo + cells, jitter=0.2, seed=seed + g)
        st = scenes.make_state(x, mass, vol, kind, group=g)
        T.perturb_state(st, kind, 1.0 / res, seed + 17 * g, 0.02, 0.5)
        if kind in (scenes.MAT_SAND,):
            st["ps"] = (st["ps"] + 2e-3 * (1 + g)).astype(np.float32)
        parts.append(st)
        kinds.append(kind)
        prms.append(scenes.material_params(kind, **kw))
    st = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    st["group"] = st["group"].astype(np.int32)
    planes = np.array([[0.0, 1.0, 0.0, -9.6]], np.float32)
    scene = dict(res=(res, res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0, 0.0), particle_gravity=1, mat_kind=np.array(kinds, np.int32),
                 mat_params=np.array(prms, np.float32), planes=planes, friction=0.4)
    return scene, st


def make_pool(st, L, kinds, seed=0, spare=5):
    """`st` in a pool of noise: slot indices[k] holds particle k's fields at the layout's offsets, its type's scalar at its
    kind's offset; every other byte (and every spare slot) is random."""
    n = len(st["x"])
    slots = n + spare
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 256, size=(slots, L.stride), dtype=np.uint8)
    indices = rng.permutation(slots)[:n].astype(np.uint32)
    f = pool.view(np.float32).reshape(slots, L.stride // 4)
    s = indices.astype(np.int64)
    f[s, L.off_pos // 4: L.off_pos // 4 + 3] = st["x"]
    f[s, L.off_v_and_m // 4: L.off_v_and_m // 4 + 3] = st["v"]
    f[s, L.off_v_and_m // 4 + 3] = st["mass"]
    for c in range(3):
        f[s, (L.off_dg_e + c * L.col_pitch) // 4: (L.off_dg_e + c * L.col_pitch) // 4 + 3] = st["F"][:, 3 * c: 3 * c + 3]
        f[s, (L.off_apic_b + c * L.col_pitch) // 4: (L.off_apic_b + c * L.col_pitch) // 4 + 3] = st["b"][:, 3 * c: 3 * c + 3]
    f[s, L.off_vol // 4] = st["vol"]
    kind_of = np.asarray(kinds)[st["group"]]
    for k, off in zip(capi.MpmbAosLayout.SCALAR_KINDS, L.off_scalar_by_kind):
        m = kind_of == k
        if off >= 0 and m.any():
            f[s[m], off // 4] = st["ps"][m]
    return pool.reshape(-1), indices


def expected_scalars(st, L, kinds):
    """What the upload packs: the slot's scalar for a kind with an offset, else mpmb_upload_particles' default."""
    kind_of = np.asarray(kinds)[st["group"]]
    out = np.where((kind_of == scenes.MAT_SNOW) | (kind_of == scenes.MAT_WATER), 1.0, 0.0).astype(np.float32)
    for k, off in zip(capi.MpmbAosLayout.SCALAR_KINDS, L.off_scalar_by_kind):
        if off >= 0:
            out[kind_of == k] = st["ps"][kind_of == k]
    return out


def engine(scene, res=RES):
    e = capi.Engine(res, 1.0 / res, scene["dt"], gravity=scene["gravity"])
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    return e


def test_mixed_pool_round_trips_byte_for_byte():
    scene, st = mixed_scene()
    L = reference_layout()
    kinds = scene["mat_kind"]
    pool, indices = make_pool(st, L, kinds, seed=1)
    e = engine(scene)
    try:
        before, idx0 = pool.copy(), indices.copy()
        e.upload_aos(pool, indices, L, group=st["group"])
        got = e.download()
        assert np.array_equal(got["id"], np.arange(len(st["x"])))
        assert np.array_equal(got["ps"], expected_scalars(st, L, kinds))
        assert np.array_equal(got["group"], st["group"]) and np.array_equal(got["x"], st["x"])
        assert e.download_aos(pool, indices, L) == len(st["x"])
        assert np.array_equal(pool, before) and np.array_equal(indices, idx0)
        # the download writes at the offsets of the upload's group kinds, whatever mpmb_set_material does in between
        e.upload_aos(pool, indices, L, group=st["group"])
        e.set_material(0, scenes.MAT_WATER, scenes.material_params(scenes.MAT_WATER))     # sand -> water
        e.set_material(3, scenes.MAT_SAND, scenes.material_params(scenes.MAT_SAND))       # water -> sand
        e.set_material(4, scenes.MAT_SNOW, scenes.material_params(scenes.MAT_SNOW))       # linear -> snow
        assert e.download_aos(pool, indices, L) == len(st["x"])
        assert np.array_equal(pool, before) and np.array_equal(indices, idx0)
    finally:
        e.close()


def test_absent_kind_offsets_take_the_upload_defaults():
    """An entry of -1 is a type without its scalar in the slot: snow and water start at Jp = j = 1, sand and visco at 0, and
    nothing is written back for them."""
    scene, st = mixed_scene()
    L = reference_layout()
    full = list(L.off_scalar_by_kind)
    L.set_scalar_offsets({scenes.MAT_VISCO: full[3]})          # only visco keeps its scalar
    kinds = scene["mat_kind"]
    pool, indices = make_pool(st, L, kinds, seed=2)
    e = engine(scene)
    try:
        before = pool.copy()
        e.upload_aos(pool, indices, L, group=st["group"])
        ps = e.download()["ps"]
        kind_of = kinds[st["group"]]
        assert np.all(ps[(kind_of == scenes.MAT_SNOW) | (kind_of == scenes.MAT_WATER)] == 1.0)
        assert np.all(ps[kind_of == scenes.MAT_SAND] == 0.0)
        assert np.array_equal(ps[kind_of == scenes.MAT_VISCO], st["ps"][kind_of == scenes.MAT_VISCO])
        assert e.download_aos(pool, indices, L) == len(st["x"])
        assert np.array_equal(pool, before)
    finally:
        e.close()


def test_bad_per_kind_layouts_are_refused_and_change_nothing():
    scene, st = mixed_scene()
    L = reference_layout()
    kinds = scene["mat_kind"]
    pool, indices = make_pool(st, L, kinds, seed=3)
    e = engine(scene)
    try:
        e.upload_aos(pool, indices, L, group=st["group"])
        resident = e.download()
        before = pool.copy()
        bad = []
        for field, k, v in [("off_scalar", None, 200), ("by_kind", 2, 218), ("by_kind", 0, 0), ("by_kind", 1, L.stride - 2),
                            ("by_kind", 3, L.stride), ("by_kind", 1, -8)]:
            B = capi.MpmbAosLayout.from_buffer_copy(L)
            if field == "off_scalar":
                B.off_scalar = v
            else:
                B.off_scalar_by_kind[k] = v
            bad.append(B)
        sub = {kk: v[: len(st["x"]) // 2] for kk, v in st.items()}
        pool2, idx2 = make_pool(sub, L, kinds, seed=4)
        for B in bad:
            with pytest.raises(capi.MpmbError) as ex:
                e.upload_aos(pool2, idx2, B, group=sub["group"])
            assert ex.value.code == -1
            with pytest.raises(capi.MpmbError) as ex:
                e.download_aos(pool, indices.copy(), B)
            assert ex.value.code == -1
            assert np.array_equal(pool, before)
            now = e.download()
            assert all(np.array_equal(now[kk], resident[kk]) for kk in resident)
        # per-kind scalars need the group kinds of an AoS upload of the resident set
        e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
        with pytest.raises(capi.MpmbError) as ex:
            e.download_aos(pool, indices.copy(), L)
        assert ex.value.code == -4
        assert np.array_equal(pool, before)
    finally:
        e.close()


def _by_type(pa, pb, ids, kind_of, tol_x, F=True):
    for k in np.unique(kind_of[ids]):
        m = ids[kind_of[ids] == k]
        assert np.abs(pa["x"][m] - pb["x"][m]).max() <= tol_x, k
        assert np.abs(pa["v"][m] - pb["v"][m]).max() <= 2e-4 * np.abs(pa["v"][m]).max(), k
        assert np.abs(pa["b"][m] - pb["b"][m]).max() <= 5e-4 * np.abs(pa["b"][m]).max(), k
        if F and k != scenes.MAT_WATER:
            assert np.abs(pa["F"][m] - pb["F"][m]).max() <= 5e-5, k
        from tests import common as T
        assert T.ps_err(pa["ps"][m], pb["ps"][m]) <= (1e-3 if k == scenes.MAT_VISCO else 5e-5), k


def run_dropin_mixed(lib_path, tmp_path, nsub=12):
    """The reference's MPM<3> object with all eight types (sand and snow twice) steps by itself (A) and through the C-ABI (B);
    both go on with its own substep() and write_partio, then B routes again with the scalars it has evolved."""
    from oracle import pyoracle_mixed as M
    from taichi_mpm_b200 import bgeo
    scene, st = mixed_scene()
    st["x"][0] = [6.5 / 32, 0.5, 0.5]                       # one particle in the deletion band
    kind_of = scene["mat_kind"][st["group"]]
    a, b = M.MixedRefSolver(scene, st), M.MixedRefSolver(scene, st)
    try:
        na, nb = a.substep(nsub), b.substep_via_mpmb(lib_path, nsub)
        pa, pb = a.particles(), b.particles()
        ids = pa["alive_ids"]
        assert na == nb == len(st["x"]) - 1 and np.array_equal(ids, pb["alive_ids"])
        moved = {k: np.abs(pa["ps"][ids] - st["ps"][ids])[kind_of[ids] == k].max() for k in (scenes.MAT_SAND, scenes.MAT_SNOW, scenes.MAT_WATER)}
        assert min(moved.values()) > 1e-6, moved                 # the scalars evolved: the download wrote them
        _by_type(pa, pb, ids, kind_of, 2e-6)
        assert a.substep(3) == b.substep(3) == na
        qa, qb = a.particles(), b.particles()
        assert np.abs(qa["x"][ids] - qb["x"][ids]).max() <= 3e-6
        fa, fb = tmp_path / "a.bgeo", tmp_path / "b.bgeo"
        a.write_partio(fa); b.write_partio(fb)
        xa, aa = bgeo.read_bgeo(str(fa))
        xb, ab = bgeo.read_bgeo(str(fb))
        assert np.array_equal(dict((n, v) for n, _, v in aa)["index"], dict((n, v) for n, _, v in ab)["index"])
        assert np.abs(xa - xb).max() <= 3e-6
        # route again: the re-upload reads the scalars the reference's own substeps evolved
        assert a.substep(4) == b.substep_via_mpmb(lib_path, 4) == na
        ra, rb = a.particles(), b.particles()
        assert np.array_equal(ra["alive_ids"], rb["alive_ids"])
        _by_type(ra, rb, ids, kind_of, 4e-6)
    finally:
        a.close(); b.close()


def test_reference_solver_steps_a_mixed_pool_through_libmpmb(tmp_path):
    from oracle import pyoracle_mixed as M
    if not M.ref_available():
        pytest.skip("reference build (oracle/_ref) not available")
    capi.lib()
    run_dropin_mixed(capi.lib_path(), tmp_path)


def run_async_mixed(lib_path, pair, steps=2):
    """The reference's AsyncMPM<3> scheduler on a pool of two types (one group each): A on its own substep, B with every substep
    routed to one libmpmb engine.  Same decisions, states to run_async's bounds."""
    from oracle import pyoracle_mixed as M
    from tests import common as T
    groups = [(k, {}) for k in pair]
    scene, st = mixed_scene(groups, cells=4, seed=5)
    st["v"][:] = 0
    st["v"][st["x"][:, 0] > 0.35, 0] = 10.0                  # a fast part: its blocks step on a finer level
    sand = scenes.MAT_SAND in pair
    unit = 5e-6 if sand else 2.5e-5
    kw = dict(unit_delta_t=unit, max_units=64, cfl_dt_mul=0.1)
    a, b = M.MixedRefAsyncSolver(scene, st, **kw), M.MixedRefAsyncSolver(scene, st, **kw)
    try:
        b.route_through(lib_path)
        keys = ("alive", "update_counter", "current_t_int", "min_level", "max_level")
        for _ in range(steps):
            ra, rb = a.step(80 * unit), b.step(80 * unit)
            assert {k: ra[k] for k in keys} == {k: rb[k] for k in keys}
        assert ra["min_level"] < ra["max_level"] and rb["routed_substeps"] > 5 and ra["routed_substeps"] == 0
        pa, pb = a.particles(), b.particles()
        m = pa["alive"].astype(bool)
        assert np.array_equal(pa["alive"], pb["alive"]) and (~m).sum() < 50
        assert np.abs(pa["x"] - pb["x"])[m].max() <= 2e-6
        assert np.abs(pa["v"] - pb["v"])[m].max() <= 2e-5 * np.abs(pa["v"]).max()
        assert np.abs(pa["F"] - pb["F"])[m].max() <= 5e-5 and T.ps_err(pa["ps"][m], pb["ps"][m]) <= 5e-5
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("pair", [(scenes.MAT_SAND, scenes.MAT_ELASTIC), (scenes.MAT_SNOW, scenes.MAT_WATER)], ids=["sand_elastic", "snow_water"])
def test_reference_asyncmpm_routes_a_mixed_pool_through_libmpmb(pair):
    from oracle import pyoracle_mixed as M
    if not M.ref_available():
        pytest.skip("reference build (oracle/_ref) not available")
    capi.lib()
    run_async_mixed(capi.lib_path(), pair)


@pytest.mark.needs_cuda
def test_million_particle_mixed_pool():
    """1 M particles, four types in four blocks of 32^3 cells: the byte round trip, then one substep after mpmb_upload_aos equal
    bit for bit to one substep after mpmb_upload_particles of the same particles, groups and scalars."""
    from tests import common as T
    res = 128
    groups = [(scenes.MAT_SAND, {}), (scenes.MAT_SNOW, {}), (scenes.MAT_WATER, {}), (scenes.MAT_VISCO, {})]
    parts = []
    for g, (kind, _) in enumerate(groups):
        lo = np.array([16 + 48 * (g % 2), 10, 16 + 48 * (g // 2)])
        x, mass, vol = scenes.lattice_block(res, lo, lo + 32, jitter=0.2, seed=40 + g)
        st = scenes.make_state(x, mass, vol, kind, group=g)
        T.perturb_state(st, kind, 1.0 / res, 50 + g, 0.02, 0.5)
        parts.append(st)
    st = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    st["group"] = st["group"].astype(np.int32)
    n = len(st["x"])
    assert n == 4 * 32 ** 3 * 8
    scene = dict(dt=2e-5, gravity=(0.0, -10.0, 0.0), mat_kind=np.array([k for k, _ in groups], np.int32),
                 mat_params=np.array([scenes.material_params(k) for k, _ in groups], np.float32))
    L = reference_layout()
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=6, spare=1000)
    before, idx0 = pool.copy(), indices.copy()
    a, b = engine(scene, res), engine(scene, res)
    try:
        a.upload_aos(pool, indices, L, group=st["group"])
        assert a.download_aos(pool, indices, L) == n
        assert np.array_equal(pool, before) and np.array_equal(indices, idx0)
        a.upload_aos(pool, indices, L, group=st["group"])
        b.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
        a.substep(1); b.substep(1)
        ga, gb = a.download(), b.download()
        for k in ga:
            assert np.array_equal(ga[k].view(np.uint8), gb[k].view(np.uint8)), k
    finally:
        a.close(); b.close()
