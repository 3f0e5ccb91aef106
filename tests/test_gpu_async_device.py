"""AsyncMPM's pools on the device (mpmb_async_*, SURVEY §8f row 3) against the host pools of the same scheduler: identical
scheduler decisions after every step and bitwise-equal pools (order, every field, id and block).  The host pools run on the same
engine with its mpmb_async_* calls hidden, so that both sides execute the same substeps; tests/test_async_host.py and
tests/test_gpu_async.py compare the scheduler with the reference's own AsyncMPM<3>."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as O
from taichi_mpm_b200 import async_mpm, capi, scenes
from tests import common as T

pytestmark = pytest.mark.gpu

_Engine = capi.Engine
NAMES = {scenes.MAT_SNOW: "snow", scenes.MAT_WATER: "water", scenes.MAT_SAND: "sand", scenes.MAT_ELASTIC: "elastic",
         scenes.MAT_VON_MISES: "von_mises", scenes.MAT_VISCO: "visco", scenes.MAT_JELLY: "jelly"}
FIELDS = ("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group")


class HostPoolsEngine:
    """The device engine without its mpmb_async_* calls: AsyncMPM then keeps its pools on the host (test-only wrapper)."""

    def __init__(self, *a, **kw):
        self._e = _Engine(*a, **kw)

    def __getattr__(self, name):
        if name.startswith("async_"):
            raise AttributeError(name)
        return getattr(self._e, name)


def _model(monkeypatch, host, **kw):
    monkeypatch.setattr(capi, "Engine", HostPoolsEngine if host else _Engine)
    m = async_mpm.AsyncMPM(res=(32, 32, 32), **kw)
    monkeypatch.setattr(capi, "Engine", _Engine)
    assert m._device_pools == (not host)
    return m


def _pair(monkeypatch, kind):
    """Host-pool and device-pool models of one scene: a block whose fast half takes a finer time level (cfl_dt_mul = 0.1)."""
    scene, st = T.perturbed_scene(kind, res=32, cells=8, seed=7, strain=0.0, vel=0.0, with_floor=False)
    st["v"][:] = 0
    st["v"][st["x"][:, 0] > 0.55, 0] = 10.0
    unit = 2.5e-5 if kind == scenes.MAT_SNOW else 5e-6
    kw = dict(base_delta_t=unit, unit_delta_t=unit, max_units=64, cfl_dt_mul=0.1, gravity=scene["gravity"])
    ms = []
    for host in (True, False):
        m = _model(monkeypatch, host, **kw)
        m.add_particles(type=NAMES[kind], positions=st["x"], density=400.0)
        for k in ("v", "mass", "vol", "F", "b", "ps"):
            m.pool[k][:] = st[k]
        ms.append(m)
    return unit, ms[0], ms[1]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same_pools(a, b):
    for pa, pb in zip(a.pools(), b.pools()):
        assert len(pa["id"]) == len(pb["id"])
        for k in FIELDS:
            assert np.array_equal(_bits(pa[k]), _bits(pb[k])), k


def _lockstep(unit, mh, md, steps, asynchronous=True):
    for _ in range(steps):
        mh.step(80 * unit)
        md.step(80 * unit)
        assert mh.scheduler_stats() == md.scheduler_stats()
    assert_same_pools(mh, md)
    s = md.scheduler_stats()
    assert s["update_counter"] > 0
    assert s["min_level"] < s["max_level"] or not asynchronous       # several time levels at once


@pytest.mark.parametrize("kind", [scenes.MAT_SNOW, scenes.MAT_SAND, scenes.MAT_WATER])
def test_device_pools_equal_host_pools_bit_for_bit(kind, monkeypatch):
    unit, mh, md = _pair(monkeypatch, kind)
    _lockstep(unit, mh, md, steps=2, asynchronous=kind != scenes.MAT_WATER)   # water's stiffness limit keeps one level here
    assert mh.num_particles() == md.num_particles()
    ph, pd = mh.get_particles(), md.get_particles()
    for k in ph:
        assert np.array_equal(_bits(ph[k]), _bits(pd[k])), k


def test_device_pools_through_deletions_and_level_changes(monkeypatch):
    # eight steps: the fast half runs into the deletion band, levels regroup every step
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    _lockstep(unit, mh, md, steps=8)
    assert md.scheduler_stats()["pool_entries"] < 3900


def test_add_particles_after_the_first_step_appends_to_the_device_pool(monkeypatch):
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    _lockstep(unit, mh, md, steps=1)
    for m in (mh, md):
        m.add_particles(type="snow", benchmark_block=((20, 20, 12), (23, 23, 15)), initial_velocity=(0.0, -3.0, 0.0))
    assert mh.num_particles() == md.num_particles() and md._on_device
    assert_same_pools(mh, md)
    _lockstep(unit, mh, md, steps=2)


def _records(rng, ids, group=0):
    n = len(ids)
    X = rng.uniform(8.0, 24.0, size=(n, 3)).astype(np.float32)
    F = (np.eye(3, dtype=np.float32).reshape(1, 9) + rng.normal(size=(n, 9)).astype(np.float32) * 0.01).astype(np.float32)
    return dict(x=(X / np.float32(32)).astype(np.float32), v=rng.normal(size=(n, 3)).astype(np.float32), F=F,
                b=(rng.normal(size=(n, 9)) * 1e-4).astype(np.float32), mass=np.full(n, 6e-6, np.float32), vol=np.full(n, 1.5e-8, np.float32),
                ps=np.ones(n, np.float32), group=np.full(n, group, np.int32), id=np.asarray(ids, np.int64))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_async_advance_against_the_host_advance(monkeypatch, seed):
    # hand-built pools (ids in both the pool and the backup, duplicates inside the pool) and random block flags: the gathered
    # set (the engine's particles after the substep, by engine id) and both pools equal the host advance's
    rng = np.random.default_rng(seed)
    kw = dict(base_delta_t=2.5e-5, unit_delta_t=2.5e-5, max_units=64)
    mh, md = _model(monkeypatch, True, **kw), _model(monkeypatch, False, **kw)
    for m in (mh, md):
        m.add_particles(type="snow", benchmark_block=((12, 12, 12), (13, 13, 13)))    # registers the material as group 0
    pool = _records(rng, np.concatenate([np.arange(600), rng.choice(600, 50, replace=False)]))
    backup = _records(rng, np.concatenate([rng.choice(600, 300, replace=False), np.arange(600, 700)]))
    for m in (mh, md):
        m.pool = {k: v.copy() for k, v in pool.items()}
        m.backup = {k: v.copy() for k, v in backup.items()}
        m.pool["block"], m.backup["block"] = m._block_of(pool["x"]), m._block_of(backup["x"])
    md._pools_to_device()
    assert_same_pools(mh, md)
    for it in range(3):
        fl = rng.integers(0, 32, size=md.nb).astype(np.uint8)
        masks = [(fl & bit) != 0 for bit in (capi.ASYNC_SMALLER, capi.ASYNC_EQUAL, capi.ASYNC_LARGER, capi.ASYNC_SWAP, capi.ASYNC_CLEAR)]
        dt = 2.5e-5 * (1 << it)
        n_host = mh._advance_host(*masks, dt)
        n_dev = md.engine.async_advance(fl, dt)
        assert n_host == n_dev > 0
        gh, gd = mh.engine.download(), md.engine.download()      # engine id = gather index on both sides
        for k in gh:
            assert np.array_equal(_bits(gh[k]), _bits(gd[k])), k
        assert_same_pools(mh, md)


def _one_per_block(kind, rng):
    bx, by, bz = np.meshgrid(np.arange(2, 6), np.arange(2, 6), np.arange(1, 3), indexing="ij")
    X = np.stack([4 * bx + 1.5, 4 * by + 1.5, 8 * bz + 1.5], -1).reshape(-1, 3).astype(np.float32)
    n = len(X)
    F = (np.eye(3)[None] + rng.normal(size=(n, 3, 3)) * 0.05).astype(np.float32).reshape(n, 9)
    ps = {scenes.MAT_SNOW: 1 + rng.normal(size=n) * 0.05, scenes.MAT_WATER: 1 + rng.normal(size=n) * 0.03}.get(kind, np.zeros(n)).astype(np.float32)
    v = (rng.normal(size=(n, 3)) * 2).astype(np.float32)
    return X / np.float32(32), F, ps, v


@pytest.mark.parametrize("kind", [scenes.MAT_SNOW, scenes.MAT_WATER, scenes.MAT_SAND, scenes.MAT_ELASTIC, scenes.MAT_VON_MISES, scenes.MAT_VISCO])
def test_block_limits_are_allowed_dt_per_particle(kind, monkeypatch):
    rng = np.random.default_rng(kind)
    x, F, ps, v = _one_per_block(kind, rng)
    m = _model(monkeypatch, False, base_delta_t=1e-5, unit_delta_t=1e-5)
    m.add_particles(type=NAMES[kind], positions=x)
    assert len(m.pool["id"]) == len(x)
    m.pool["F"][:], m.pool["ps"][:], m.pool["v"][:] = F, ps, v
    m._pools_to_device()
    blk, mn, mx = m.engine.async_block_limits(True)
    p = m.pool if m.pool is not None else m.pools()[0]
    lin = (p["block"][:, 0] * m.nb[1] + p["block"][:, 1]) * m.nb[2] + p["block"][:, 2]
    o = np.argsort(lin)
    assert np.array_equal(blk, lin[o])
    kk, prm = m._groups[0]
    host = np.minimum(np.float32(0.1), async_mpm.allowed_dt(kk, prm, p["F"], p["ps"], p["mass"], p["vol"], p["v"], m.delta_x))[o]
    assert (host < 0.1).all()
    assert np.abs(mn.view(np.int32).astype(np.int64) - host.view(np.int32)).max() <= 2          # within 2 ulp of the host's
    assert np.array_equal(mx.view(np.uint32), np.maximum((p["v"].astype(np.float32) ** 2).sum(1), np.float32(1e-16))[o].view(np.uint32))
    if O.ref_particles_available():
        Fcm = np.ascontiguousarray(np.transpose(p["F"].reshape(-1, 3, 3), (0, 2, 1)).reshape(-1, 9))
        ref = np.array([O.ref_allowed_dt(kk, prm, Fcm[i], float(p["ps"][i]), float(p["mass"][i]), float(p["vol"][i]), p["v"][i], m.delta_x)
                        for i in o])
        assert np.abs(mn - np.minimum(ref, 0.1)).max() <= 2e-6 * ref.max()
    b2, n2, x2 = m.engine.async_block_limits(False)
    assert np.array_equal(b2, blk) and n2 is None and x2 is None


def test_jelly_in_the_device_pool_raises(monkeypatch):
    m = _model(monkeypatch, False, base_delta_t=1e-5, unit_delta_t=1e-5)
    m.add_particles(type="jelly", benchmark_block=((12, 12, 12), (14, 14, 14)))
    with pytest.raises(ValueError):
        m.step(1e-4)
    assert m._on_device


def test_no_particle_record_crosses_the_bus_inside_step(monkeypatch):
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    calls = []
    for name in ("upload", "download", "append", "upload_ptrs", "download_ptrs", "async_download"):
        real = getattr(md.engine, name)
        setattr(md.engine, name, (lambda real, name: lambda *a, **k: (calls.append(name), real(*a, **k))[1])(real, name))
    md.step(80 * unit)
    md.step(80 * unit)
    assert calls == []
    assert md.scheduler_stats()["update_counter"] > 0 and calls == ["async_download", "async_download"]   # outside step(): reads


def _raw(e):
    return e.L, e.h


def test_error_codes():
    nb = (C.c_int32 * 3)(16, 16, 8)
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4)
    e.set_material(0, capi.MAT_SNOW, scenes.material_params(scenes.MAT_SNOW))
    L, h = _raw(e)
    n = C.c_int64(0)
    fl = np.zeros(16 * 16 * 8, np.uint8)
    # before mpmb_async_init: MPMB_ERR_STATE (-4)
    for rc in (L.mpmb_async_add(h, 0, C.c_int64(0), None, None, None, None, None, None, None, None, None),
               L.mpmb_async_block_limits(h, 0, C.c_int64(0), C.byref(n), None, None, None),
               L.mpmb_async_advance(h, fl.ctypes.data_as(C.c_void_p), C.c_float(1e-4), C.byref(n)),
               L.mpmb_async_size(h, C.byref(n), None),
               L.mpmb_async_download(h, 0, C.c_int64(0), C.byref(n), *([None] * 10))):
        assert rc == -4
    assert L.mpmb_async_init(h, nb, C.c_float(32.0)) == 0
    # bad arguments
    assert L.mpmb_async_advance(h, None, C.c_float(1e-4), C.byref(n)) == -1
    assert L.mpmb_async_add(h, 2, C.c_int64(0), None, None, None, None, None, None, None, None, None) == -1
    assert L.mpmb_async_download(h, -1, C.c_int64(0), C.byref(n), *([None] * 10)) == -1
    rng = np.random.default_rng(3)
    rec = _records(rng, np.arange(64))
    e.async_add(0, rec)
    far = dict(rec, x=np.full((64, 3), 5.0, np.float32))                 # outside the block grid
    with pytest.raises(capi.MpmbError) as ex:
        e.async_add(0, far)
    assert ex.value.code == -1 and e.async_size() == (64, 0)
    # inside a substep
    e.upload(rec["x"], rec["v"], rec["mass"], rec["vol"])
    e.sort_particles_and_populate_grid()
    assert L.mpmb_async_advance(h, fl.ctypes.data_as(C.c_void_p), C.c_float(1e-4), C.byref(n)) == -4
    assert L.mpmb_async_size(h, C.byref(n), None) == -4
    e.rasterize()
    e.resample()
    e.close()
    # a configured capacity below the gathered set: both pools unchanged
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4, capacity=32)
    e.set_material(0, capi.MAT_SNOW, scenes.material_params(scenes.MAT_SNOW))
    e.async_init((16, 16, 8), 32.0)
    e.async_add(0, rec)
    e.async_add(1, _records(rng, np.arange(10)))
    before = [e.async_download(w) for w in (0, 1)]
    with pytest.raises(capi.MpmbError) as ex:
        e.async_advance(np.full(16 * 16 * 8, capi.ASYNC_EQUAL | capi.ASYNC_SWAP | capi.ASYNC_CLEAR, np.uint8), 1e-4)
    assert ex.value.code == -3
    after = [e.async_download(w) for w in (0, 1)]
    for a, b in zip(before, after):
        for k in a:
            assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    e.close()
    # z-slab ranks and rigid samples
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4, world=2, rank=0, tile_z0=0, tile_z1=4, migrate_capacity=1024)
    assert e.L.mpmb_async_init(e.h, nb, C.c_float(32.0)) == -4
    e.close()
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4)
    off, tri, rid = np.zeros(3, np.float32), np.zeros(9, np.float32), np.ones(1, np.int32)
    tri[3], tri[7] = 1.0, 1.0
    assert e.L.mpmb_set_rigid_samples(e.h, 2, C.c_int64(1), off.ctypes.data_as(C.c_void_p), tri.ctypes.data_as(C.c_void_p),
                                      rid.ctypes.data_as(C.c_void_p)) == 0
    assert e.L.mpmb_async_init(e.h, nb, C.c_float(32.0)) == -4
    e.close()
