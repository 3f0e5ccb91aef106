"""The 2-D drop-in (INTEGRATION.md §2): mpmb_upload_aos / mpmb_download_aos on a 2-D handle, reading and writing MPM<2>'s own
AoS pool (ParticleContainer<2> slots: pos float[2], v_and_m float[3] = (vx, vy, mass), dg_e and apic_b as two columns of two
floats `col_pitch` apart, vol, the plastic scalar).

  * byte round trip: a pool of noise comes back byte for byte from upload -> download with 0 substeps, and after substeps no
    byte outside the layout's fields has changed; with a padded layout (16-byte columns), a packed one (col_pitch 8, v_and_m
    12 bytes) and the reference's in-place one;
  * the rows are the field-wise path's: the same particles through mpmb_upload_aos and mpmb_upload_particles give
    bit-identical mpmb_download_particles after 50 substeps, with graphs and without, single-type and mixed;
  * refusals (bad layouts, a slot outside the pool, a per-kind download without an AoS upload) change nothing;
  * the reference's own MPM<2> object steps 12 substeps by itself and through the C-ABI (oracle/transfer2d_aos_ref.cpp), for
    every material and for a mixed pool, then both go on with MPM<2>::substep() and write_partio;
  * full size: bench_2d.py's 2048^2 sand column through the AoS calls against the chained fp64 2-D oracle.

tests/test_dropin_2d.py runs this file on the SIMT emulator (all but the full-size test)."""
import os

import numpy as np
import pytest

from oracle import pyoracle2d_aos as A
from taichi_mpm_b200 import capi, scenes
from tests import common as T
from tests.mpm2d_common import scene2d, state_of
from tests.test_gpu_mpm2d import KINDS, assert_parity, compare2d

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not A.ref_available(), reason="reference build (oracle/_ref) not available")
ERR_INVALID, ERR_STATE = -1, -4   # MPMB_ERR_INVALID, MPMB_ERR_STATE (include/mpmb.h)

FIELDS = ("stride", "off_pos", "off_v_and_m", "off_dg_e", "off_apic_b", "col_pitch", "off_vol", "off_scalar")
# ParticleContainer<2> of the in-place reference build (192-byte slots), offsetof() on its classes: checked against
# oracle/pyoracle2d_aos.aos_layout by test_inplace_layout_is_the_reference_build_s
INPLACE = (192, 32, 16, 40, 56, 8, 84)
INPLACE_SCALARS = {scenes.MAT_SNOW: 116, scenes.MAT_WATER: 124, scenes.MAT_SAND: 136, scenes.MAT_VISCO: 116}
LAYOUTS = {
    "padded": (160, 0, 16, 32, 64, 16, 96),   # every small vector in 16 bytes
    "packed": (60, 0, 8, 20, 36, 8, 52),      # VectorND<2, float> in 8 bytes, v_and_m in 12
    "inplace": INPLACE,
}
SCALAR_AFTER = {"padded": 100, "packed": 56}  # the single plastic scalar behind vol


def layout(name, kind=None, per_kind=False):
    """MpmbAosLayout `name` with the scalar of `kind` (single-offset mode) or every kind's (per-kind mode)."""
    L = capi.MpmbAosLayout()
    for f, v in zip(FIELDS, LAYOUTS[name]):
        setattr(L, f, int(v))
    sc = INPLACE_SCALARS if name == "inplace" else {k: SCALAR_AFTER[name] for k in capi.MpmbAosLayout.SCALAR_KINDS}
    if per_kind:
        L.set_scalar_offsets(sc)
    else:
        L.off_scalar = sc.get(kind, -1)
    return L


def field_spans(L):
    """(offset, bytes) of every field the layout names."""
    spans = [(L.off_pos, 8), (L.off_v_and_m, 12), (L.off_vol, 4)]
    spans += [(o + c * L.col_pitch, 8) for o in (L.off_dg_e, L.off_apic_b) for c in range(2)]
    if L.off_scalar >= 0:
        spans.append((L.off_scalar, 4))
    spans += [(o, 4) for o in L.off_scalar_by_kind if o > 0]
    return spans


def make_pool(st, L, kinds, seed=0, spare=7):
    """`st` in a pool of noise: slot indices[k] holds particle k's fields at the layout's offsets, its scalar at its kind's
    offset (per kind) or at off_scalar; every other byte and every spare slot is random."""
    n = len(st["x"])
    slots = n + spare
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 256, size=(slots, L.stride), dtype=np.uint8)
    indices = rng.permutation(slots)[:n].astype(np.uint32)
    f = pool.view(np.float32).reshape(slots, L.stride // 4)
    s = indices.astype(np.int64)
    f[s, L.off_pos // 4: L.off_pos // 4 + 2] = st["x"]
    f[s, L.off_v_and_m // 4: L.off_v_and_m // 4 + 2] = st["v"]
    f[s, L.off_v_and_m // 4 + 2] = st["mass"]
    for c in range(2):
        f[s, (L.off_dg_e + c * L.col_pitch) // 4: (L.off_dg_e + c * L.col_pitch) // 4 + 2] = st["F"][:, 2 * c: 2 * c + 2]
        f[s, (L.off_apic_b + c * L.col_pitch) // 4: (L.off_apic_b + c * L.col_pitch) // 4 + 2] = st["b"][:, 2 * c: 2 * c + 2]
    f[s, L.off_vol // 4] = st["vol"]
    if any(L.off_scalar_by_kind):
        kind_of = np.asarray(kinds)[st["group"]]
        for k, off in zip(capi.MpmbAosLayout.SCALAR_KINDS, L.off_scalar_by_kind):
            if off >= 0 and (kind_of == k).any():
                f[s[kind_of == k], off // 4] = st["ps"][kind_of == k]
    elif L.off_scalar >= 0:
        f[s, L.off_scalar // 4] = st["ps"]
    return pool.reshape(-1), indices


def mixed_scene2d(seed=3):
    """Sand, snow, water and visco blocks side by side on a floor (they collide), each perturbed as its type."""
    parts, kinds, prms = [], [], []
    for g, kind in enumerate((scenes.MAT_SAND, scenes.MAT_SNOW, scenes.MAT_WATER, scenes.MAT_VISCO)):
        lo = (8 + 4 * g, 9)
        sc, st = scene2d(kind, blocks=[(lo, (lo[0] + 4, 15))], seed=seed + g, **(dict(kappa=0.3) if kind == scenes.MAT_VISCO else {}))
        st["group"][:] = g
        parts.append(st)
        kinds.append(kind)
        prms.append(sc["mat_params"][0])
    st = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    st["group"] = st["group"].astype(np.int32)
    scene = dict(sc, mat_kind=np.array(kinds, np.int32), mat_params=np.array(prms, np.float32), dt=2e-5)
    return scene, st


def engine(scene, **kw):
    """A 2-D handle with the scene's materials and level set, no particles."""
    e = capi.Engine2D(scene["res"], scene["dx"], scene["dt"], scene["gravity"], scene.get("particle_gravity", 1), scene["clean_boundary"],
                      apic_damping=scene.get("apic_damping", 0.0), rpic_damping=scene.get("rpic_damping", 0.0), **kw)
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    if scene.get("planes") is not None:
        e.set_planes(scene["planes"], scene["friction"])
    return e


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_round_trip_byte_for_byte(name):
    scene, st = scene2d(scenes.MAT_SAND, seed=1)
    L = layout(name, scenes.MAT_SAND)
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=2)
    before, idx0 = pool.copy(), indices.copy()
    e = engine(scene)
    try:
        e.upload_aos(pool, indices, L)
        got = e.download()
        assert np.array_equal(got["id"], np.arange(len(st["x"])))
        for k in ("x", "v", "F", "b", "mass", "vol", "ps"):
            assert np.array_equal(got[k], st[k]), k
        assert e.download_aos(pool, indices, L) == len(st["x"])
        assert np.array_equal(pool, before) and np.array_equal(indices, idx0)
    finally:
        e.close()


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_substeps_write_only_the_layout_s_fields(name):
    scene, st = scene2d(scenes.MAT_SNOW, seed=4, vel=1.0)
    st["x"][3] = [7.2 / 32, 0.5]
    st["v"][3] = [-300.0, 0.0]     # into the band: deleted by the first G2P
    L = layout(name, scenes.MAT_SNOW)
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=5)
    before, idx0 = pool.copy(), indices.copy()
    e = engine(scene)
    try:
        e.upload_aos(pool, indices, L)
        e.substep(5)
        got = e.download()
        n = e.download_aos(pool, indices, L)
        assert n == len(st["x"]) - 1 and np.array_equal(indices[:n], np.delete(idx0, 3))
        assert np.array_equal(indices[n:], idx0[n:])      # the tail of the vector is not written
        owned = np.zeros(L.stride, bool)
        for o, b in field_spans(L):
            owned[o: o + b] = True
        p, q = pool.reshape(-1, L.stride), before.reshape(-1, L.stride)
        assert np.array_equal(p[:, ~owned], q[:, ~owned])
        assert np.array_equal(p[idx0[3]], q[idx0[3]])    # the deleted particle's slot is not written
        changed = np.setdiff1d(np.arange(len(p)), idx0)   # nor any slot outside the index vector
        assert np.array_equal(p[changed], q[changed])
        f = p.view(np.float32)
        s = indices[:n].astype(np.int64)
        assert np.array_equal(f[s, L.off_pos // 4: L.off_pos // 4 + 2], got["x"])
        assert np.array_equal(f[s, L.off_v_and_m // 4: L.off_v_and_m // 4 + 2], got["v"])
        assert np.array_equal(f[s, L.off_v_and_m // 4 + 2], got["mass"])
        assert np.array_equal(f[s, (L.off_dg_e + L.col_pitch) // 4: (L.off_dg_e + L.col_pitch) // 4 + 2], got["F"][:, 2:])
        assert np.array_equal(f[s, L.off_apic_b // 4: L.off_apic_b // 4 + 2], got["b"][:, :2])
        assert np.array_equal(f[s, L.off_scalar // 4], got["ps"])
    finally:
        e.close()


@pytest.mark.parametrize("mixed", [False, True], ids=["sand", "mixed"])
@pytest.mark.parametrize("no_graph", [False, True], ids=["graph", "no_graph"])
def test_bit_identical_to_the_field_wise_upload(no_graph, mixed):
    scene, st = mixed_scene2d() if mixed else scene2d(scenes.MAT_SAND, seed=6, vel=0.5)
    L = layout("inplace", scenes.MAT_SAND, per_kind=mixed)
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=7)
    outs = []
    for aos in (True, False):
        e = engine(scene, no_graph=no_graph)
        try:
            if aos:
                e.upload_aos(pool, indices, L, group=st["group"])
            else:
                e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
            e.substep(50)
            outs.append(e.download(sort_by_id=False))
        finally:
            e.close()
    assert len(outs[0]["id"]) > 0.9 * len(st["x"])
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), k


def _same_engine(e, ref):
    got = e.download(sort_by_id=False)
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k


def test_refusals_change_nothing():
    scene, st = scene2d(scenes.MAT_SAND, seed=8)
    L = layout("inplace", scenes.MAT_SAND)
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=9)
    e = engine(scene)
    try:
        e.upload_aos(pool, indices, L)
        e.substep(2)
        ref = e.download(sort_by_id=False)
        p0, i0 = pool.copy(), indices.copy()

        def bad(field, value):
            B = layout("inplace", scenes.MAT_SAND)
            setattr(B, field, value)
            return B
        bad_layouts = [bad("off_vol", 190), bad("off_dg_e", 192 - 12), bad("off_pos", 186), bad("col_pitch", 4), bad("off_v_and_m", 18),
                       bad("off_scalar", 190), bad("stride", 190), layout("inplace", per_kind=True)]
        bad_layouts[-1].off_scalar_by_kind[2] = 138   # sand logJp misaligned
        for B in bad_layouts:
            with pytest.raises(capi.MpmbError) as ex:
                e.upload_aos(pool, indices, B)
            assert ex.value.code == ERR_INVALID
            with pytest.raises(capi.MpmbError) as ex:
                e.download_aos(pool, indices, B)
            assert ex.value.code == ERR_INVALID
            _same_engine(e, ref)
        # a slot index outside the pool: upload and download both refuse, host pool and index vector untouched
        slots = len(pool) // L.stride
        wrong = indices.copy()
        wrong[5] = slots
        with pytest.raises(capi.MpmbError) as ex:
            e.upload_aos(pool, wrong, L)
        assert ex.value.code == ERR_INVALID
        _same_engine(e, ref)
        w0 = wrong.copy()
        with pytest.raises(capi.MpmbError) as ex:
            e.download_aos(pool, wrong, L)
        assert ex.value.code == ERR_INVALID
        assert np.array_equal(pool, p0) and np.array_equal(wrong, w0)
        _same_engine(e, ref)
        # per-kind offsets need the group kinds of an AoS upload of the resident set
        e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
        with pytest.raises(capi.MpmbError) as ex:
            e.download_aos(pool, indices, layout("inplace", per_kind=True))
        assert ex.value.code == ERR_STATE
        assert np.array_equal(pool, p0) and np.array_equal(indices, i0)
        # still usable: the same pool goes through and steps
        e.upload_aos(pool, indices, L)
        e.substep(2)
        _same_engine(e, ref)
        assert e.download_aos(pool, indices, L) == len(st["x"])
    finally:
        e.close()


# ---------------------------------------------------------------- the reference's own MPM<2> object
@needs_ref
def test_inplace_layout_is_the_reference_build_s():
    lay = A.aos_layout(-1)
    assert tuple(int(v) for v in lay[:7]) == INPLACE and lay[7] == -1
    assert dict(zip(capi.MpmbAosLayout.SCALAR_KINDS, (int(v) for v in lay[8:]))) == INPLACE_SCALARS
    for k in range(8):
        assert A.aos_layout(k)[7] == INPLACE_SCALARS.get(k, -1)


def run_dropin2d(lib_path, kind, tmp_path, nsub=12, mixed=False):
    """Two reference MPM<2> objects from the same perturbed state (one particle in the deletion band): A runs nsub substeps by
    MPM<2>::substep(), B through the C-ABI; then both go on with substep() and write_partio.  The bounds are
    tests/test_dropin.py's for MPM<3>."""
    if mixed:
        scene, st = mixed_scene2d(seed=11)
    else:
        kw = dict(strain=0.006) if kind == scenes.MAT_VON_MISES else {}
        if kind == scenes.MAT_VISCO:
            kw["kappa"] = 0.3
        scene, st = scene2d(kind, seed=9 + kind, **kw)
    st["x"][0] = [6.5 * scene["dx"], 0.5]                      # one particle in the deletion band
    a, b = A.AosRefSolver2D(scene, st), A.AosRefSolver2D(scene, st)
    try:
        na = a.substep(nsub)
        nb = b.substep_via_mpmb(lib_path, nsub)
        pa, pb = a.particles(), b.particles()
        ids = np.flatnonzero(pa["alive"])
        assert na == nb == len(st["x"]) - 1 and np.array_equal(pa["alive"], pb["alive"])
        assert np.abs(pa["x"][ids] - pb["x"][ids]).max() <= 2e-6
        assert np.abs(pa["v"][ids] - pb["v"][ids]).max() <= 2e-4 * np.abs(pa["v"][ids]).max()
        assert np.abs(pa["b"][ids] - pb["b"][ids]).max() <= 5e-4 * np.abs(pa["b"][ids]).max()
        kinds = np.asarray(scene["mat_kind"])[st["group"]][ids]
        solid = kinds != scenes.MAT_WATER
        if solid.any():
            assert np.abs(pa["F"][ids][solid] - pb["F"][ids][solid]).max() <= 5e-5
        visco = kinds == scenes.MAT_VISCO
        assert T.ps_err(pa["ps"][ids][~visco], pb["ps"][ids][~visco]) <= 5e-5
        if visco.any():
            assert T.ps_err(pa["ps"][ids][visco], pb["ps"][ids][visco]) <= 1e-3
        # the pool is a valid reference state again: both go on with MPM<2>::substep and dump a frame with write_partio
        assert a.substep(3) == b.substep(3) == na
        qa, qb = a.particles(), b.particles()
        assert np.array_equal(qa["alive"], qb["alive"])
        assert np.abs(qa["x"][ids] - qb["x"][ids]).max() <= 3e-6
        fa, fb = tmp_path / "a.bgeo", tmp_path / "b.bgeo"
        a.write_partio(fa)
        b.write_partio(fb)
    finally:
        a.close()
        b.close()
    from taichi_mpm_b200 import bgeo
    xa, aa = bgeo.read_bgeo(str(fa))
    xb, ab = bgeo.read_bgeo(str(fb))
    assert np.array_equal(dict((n, v) for n, _, v in aa)["index"], dict((n, v) for n, _, v in ab)["index"])
    assert np.abs(xa - xb).max() <= 3e-6


@needs_ref
@pytest.mark.parametrize("name,kind", KINDS, ids=[k[0] for k in KINDS])
def test_reference_solver_steps_through_the_c_abi(name, kind, tmp_path):
    run_dropin2d(capi.lib_path(), kind, tmp_path)


@needs_ref
def test_reference_solver_steps_a_mixed_pool_through_the_c_abi(tmp_path):
    run_dropin2d(capi.lib_path(), None, tmp_path, mixed=True)


# ---------------------------------------------------------------- full size
@pytest.mark.skipif(bool(os.environ.get("MPMB_SIMT")), reason="4.19 M particles: GPU only")
def test_full_size_column_through_the_aos_calls():
    """bench_2d.py's 2048^2 sand column (4.19 M particles) in a pool of 192-byte slots: 3 substeps through the AoS calls
    against 3 chained substeps of the fp64 oracle (survivors, centre of mass, momentum at the bounds of
    test_gpu_mpm2d.test_collapse_chained_against_the_chained_oracle), then one more substep compared stage by stage."""
    import bench_2d as B
    from oracle import pyoracle2d as O
    res = 2048
    st, dt = B.column(res)
    scene = dict(res=(res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0), particle_gravity=1, clean_boundary=1, apic_damping=0.0,
                 rpic_damping=0.0, mat_kind=np.array([scenes.MAT_SAND], np.int32), mat_params=scenes.material_params(scenes.MAT_SAND)[None],
                 friction=0.4, planes=np.array([[0.0, 1.0, 0.0, -float(B.FLOOR)]], np.float32))
    scene["sdf"] = scenes.planes_sdf2d(scene["res"], scene["planes"])
    scene["route"] = ("planes", scene["planes"])
    st["group"] = st["group"].astype(np.int32)
    L = layout("inplace", scenes.MAT_SAND)
    pool, indices = make_pool(st, L, scene["mat_kind"], seed=12, spare=0)
    e = engine(scene)
    try:
        e.upload_aos(pool, indices, L)
        e.substep(3)
        n = e.download_aos(pool, indices, L)
        ref = st
        for _ in range(3):
            ref = O.substep2d(scene, ref, np.float64, want_grids=False)[0]
        alive = ref["alive"].astype(bool)
        got = e.download()
        assert n == alive.sum() == len(got["id"]) and np.array_equal(got["id"], np.nonzero(alive)[0])
        m = got["mass"].astype(np.float64)
        com_g, com_o = (m[:, None] * got["x"]).sum(0) / m.sum(), (m[:, None] * ref["x"][alive]).sum(0) / m.sum()
        mom_g, mom_o = (m[:, None] * got["v"]).sum(0), (m[:, None] * ref["v"][alive]).sum(0)
        assert np.abs(com_g - com_o).max() < 2e-5
        assert np.abs(mom_g - mom_o).max() <= 2e-3 * max(np.abs(mom_o).max(), m.sum() * 0.01)
        # the pool holds what the engine holds
        f = pool.reshape(-1, L.stride).view(np.float32)
        s = indices[:n].astype(np.int64)
        assert np.array_equal(f[s, L.off_pos // 4: L.off_pos // 4 + 2], got["x"])
        err, _, _ = compare2d(e, scene, state_of(got), ids=got["id"])
        assert_parity(err)
    finally:
        e.close()
