"""AsyncMPM's block scheduler on the device (mpmb_async_schedule / mpmb_async_advance_level) against the numpy scheduler over
the same device pools: after every scheduler iteration the block state (level, local_min, particle_t, backup_t) and the two
level bounds are equal bit for bit, after every advance the gathered count and both pools.  The numpy side runs on the same
engine with the scheduler calls hidden, so that both sides execute the same substeps; tests/test_gpu_async_device.py compares
the device pools with host pools."""
import ctypes as C

import numpy as np
import pytest

from taichi_mpm_b200 import async_mpm, capi, scenes
from tests import common as T

pytestmark = pytest.mark.gpu

_Engine = capi.Engine
NAMES = {scenes.MAT_SNOW: "snow", scenes.MAT_WATER: "water", scenes.MAT_SAND: "sand"}
FIELDS = ("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group")
STATE = ("level", "local_min", "particle_t", "backup_t")
SCHED_CALLS = ("async_schedule", "async_advance_level", "async_block_state")


class HostSchedEngine:
    """The device engine without its block-scheduler calls: AsyncMPM keeps the pools on the device and schedules with numpy
    (test-only wrapper)."""

    def __init__(self, *a, **kw):
        self._e = _Engine(*a, **kw)

    def __getattr__(self, name):
        if name in SCHED_CALLS:
            raise AttributeError(name)
        return getattr(self._e, name)


def _model(monkeypatch, device_sched, **kw):
    monkeypatch.setattr(capi, "Engine", _Engine if device_sched else HostSchedEngine)
    m = async_mpm.AsyncMPM(res=(32, 32, 32), **kw)
    monkeypatch.setattr(capi, "Engine", _Engine)
    assert m._device_pools and m._device_sched == device_sched
    return m


def _two_bands(x):
    v = np.zeros((len(x), 3), np.float32)
    v[x[:, 0] > 0.55, 0] = 10.0
    return v


def _three_bands(x):
    """x velocity by the particle's block row in y: 10 (level 8), 6 (level 16) and 0 (snow's strength limit is above 32
    units: level max_units = 32)."""
    by = (x[:, 1].astype(np.float32) * np.float32(32.0) - np.float32(0.5)).astype(np.int32) >> 2
    v = np.zeros((len(x), 3), np.float32)
    v[by <= 2, 0] = 10.0
    v[by == 3, 0] = 6.0
    return v


def _pair(monkeypatch, kind, velocity=_two_bands, max_units=64):
    """Numpy-scheduled and device-scheduled models of one scene (cfl_dt_mul = 0.1: fast blocks take finer levels)."""
    scene, st = T.perturbed_scene(kind, res=32, cells=8, seed=7, strain=0.0, vel=0.0, with_floor=False)
    st["v"][:] = velocity(st["x"])
    unit = 2.5e-5 if kind == scenes.MAT_SNOW else 5e-6
    kw = dict(base_delta_t=unit, unit_delta_t=unit, max_units=max_units, cfl_dt_mul=0.1, gravity=scene["gravity"])
    ms = []
    for device_sched in (False, True):
        m = _model(monkeypatch, device_sched, **kw)
        m.add_particles(type=NAMES[kind], positions=st["x"], density=400.0)
        for k in ("v", "mass", "vol", "F", "b", "ps"):
            m.pool[k][:] = st[k]
        ms.append(m)
    return unit, ms[0], ms[1]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _same_pools(a, b):
    for pa, pb in zip(a, b):
        assert len(pa["id"]) == len(pb["id"])
        for k in FIELDS:
            assert np.array_equal(_bits(pa[k]), _bits(pb[k])), k


def _same_state(a, b):
    for k in STATE:
        assert a[k].dtype == b[k].dtype == np.int64 and a[k].shape == b[k].shape
        assert np.array_equal(a[k], b[k]), k


def _logged(m):
    """Records the block state after every scheduler iteration and the gathered count and pools after every advance."""
    log = []
    update, advance = m.update_dt_limits, m.advance

    def logged_update():
        update()
        log.append(("iteration", m.current_t_int, m.min_delta_t_int, m.max_delta_t_int, m.block_state()))

    def logged_advance(limit):
        n0 = m.update_counter
        advance(limit)
        log.append(("advance", m.current_t_int, limit, m.update_counter - n0, m.pools()))
    m.update_dt_limits, m.advance = logged_update, logged_advance
    return log


def _lockstep(unit, mh, md, steps):
    """Steps both models; returns the device side's (min, max, levels of occupied blocks) of every iteration."""
    lh, ld = _logged(mh), _logged(md)
    seen = []
    for _ in range(steps):
        mh.step(80 * unit)
        md.step(80 * unit)
        assert len(lh) == len(ld) > 0
        for a, b in zip(lh, ld):
            assert a[:4] == b[:4]
            if a[0] == "iteration":
                _same_state(a[4], b[4])
                seen.append((b[2], b[3], b[4]["level"]))
            else:
                _same_pools(a[4], b[4])
        lh.clear()
        ld.clear()
        assert mh.scheduler_stats() == md.scheduler_stats()
    del mh.update_dt_limits, mh.advance, md.update_dt_limits, md.advance
    return seen


@pytest.mark.parametrize("kind", [scenes.MAT_SNOW, scenes.MAT_SAND, scenes.MAT_WATER])
def test_device_schedule_equals_numpy_schedule_bit_for_bit(kind, monkeypatch):
    unit, mh, md = _pair(monkeypatch, kind)
    _lockstep(unit, mh, md, steps=2)
    s = md.scheduler_stats()
    assert s["update_counter"] > 0
    assert s["min_level"] < s["max_level"] or kind == scenes.MAT_WATER     # water's stiffness limit keeps one level here
    ph, pd = mh.get_particles(), md.get_particles()
    for k in ph:
        assert np.array_equal(_bits(ph[k]), _bits(pd[k])), k


def test_three_levels_at_once_and_max_units(monkeypatch):
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW, _three_bands, max_units=32)
    occupied = np.zeros(md.nb, bool)
    p = md.pool
    occupied[p["block"][:, 0], p["block"][:, 1], p["block"][:, 2]] = True
    seen = _lockstep(unit, mh, md, steps=3)
    assert max(len(np.unique(lv[occupied])) for _, _, lv in seen) >= 3
    assert any(hi == md.max_units == 32 for _, hi, _ in seen)


def test_device_schedule_through_deletions_and_level_changes(monkeypatch):
    # eight steps: the fast half runs into the deletion band, levels regroup every step
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    _lockstep(unit, mh, md, steps=8)
    assert md.scheduler_stats()["pool_entries"] < 3900


def test_add_particles_after_the_first_step(monkeypatch):
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    _lockstep(unit, mh, md, steps=1)
    for m in (mh, md):
        m.add_particles(type="snow", benchmark_block=((20, 20, 12), (23, 23, 15)), initial_velocity=(0.0, -3.0, 0.0))
    assert mh.num_particles() == md.num_particles()
    _same_pools(mh.pools(), md.pools())
    _lockstep(unit, mh, md, steps=2)


def test_step_makes_one_schedule_call_per_iteration_and_one_advance_call_per_level_turn(monkeypatch):
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    counts = {"iterations": 0, "advances": 0}
    update, advance = mh.update_dt_limits, mh.advance

    def counted_update():
        counts["iterations"] += 1
        update()

    def counted_advance(limit):
        counts["advances"] += 1
        advance(limit)
    mh.update_dt_limits, mh.advance = counted_update, counted_advance
    md._pools_to_device()                    # async_init and the first async_add happen before step() here
    calls = []
    for name in [n for n in dir(md.engine) if not n.startswith("_")]:
        real = getattr(md.engine, name)
        if callable(real):
            setattr(md.engine, name, (lambda real, name: lambda *a, **k: (calls.append(name), real(*a, **k))[1])(real, name))
    for _ in range(2):
        mh.step(80 * unit)
        md.step(80 * unit)
    assert counts["advances"] >= counts["iterations"] > 0      # every iteration advances its finest level at least
    assert calls.count("async_schedule") == counts["iterations"]
    assert calls.count("async_advance_level") == counts["advances"]
    assert set(calls) == {"async_schedule", "async_advance_level"}, sorted(set(calls))
    _same_pools(mh.pools(), md.pools())


def _run_until_error(m, unit, steps, error):
    """Steps until `error` is raised; returns (the number of scheduler iterations, block state and level bounds before the
    failing one, after it)."""
    its, before = [0], [None]
    update = m.update_dt_limits

    def counted_update():
        its[0] += 1
        before[0] = (m.block_state(), m.min_delta_t_int, m.max_delta_t_int)
        update()
    m.update_dt_limits = counted_update
    with pytest.raises(error):
        for _ in range(steps):
            m.step(80 * unit)
    return its[0], before[0], (m.block_state(), m.min_delta_t_int, m.max_delta_t_int)


@pytest.mark.parametrize("what", ["nan_velocity", "jelly"])
def test_schedule_errors_at_the_numpy_iteration_with_the_state_unchanged(what, monkeypatch):
    # one step, then particles land in a block of their own: a NaN velocity makes its limit NaN when it is due
    # (RuntimeError); jelly has no limit (ValueError) once any occupied block is due
    unit, mh, md = _pair(monkeypatch, scenes.MAT_SNOW)
    _lockstep(unit, mh, md, steps=1)
    kw = dict(type="snow", initial_velocity=(float("nan"), 0.0, 0.0)) if what == "nan_velocity" else dict(type="jelly")
    error = RuntimeError if what == "nan_velocity" else ValueError
    res = []
    for m in (mh, md):
        n = m.num_particles()
        m.add_particles(benchmark_block=((8, 22, 8), (9, 23, 9)), **kw)     # 7 cells from the walls: not dropped
        assert m.num_particles() == n + 8
        res.append(_run_until_error(m, unit, steps=4, error=error))
    (ih, bh, ah), (id_, bd, ad) = res
    assert ih == id_
    for before, after in ((bh, ah), (bd, ad)):
        _same_state(before[0], after[0])
        assert before[1:] == after[1:]
    _same_state(ah[0], ad[0])
    assert ah[1:] == ad[1:]


def test_jelly_in_a_due_block_raises(monkeypatch):
    m = _model(monkeypatch, True, base_delta_t=1e-5, unit_delta_t=1e-5)
    m.add_particles(type="jelly", benchmark_block=((12, 12, 12), (14, 14, 14)))
    with pytest.raises(ValueError):
        m.step(1e-4)
    assert m._on_device and m.current_t_int == 0
    st = m.block_state()
    assert (st["level"] == 1).all() and (st["local_min"] == 1).all() and not st["particle_t"].any() and not st["backup_t"].any()


def _records(rng, n, vx=0.0):
    X = rng.uniform(8.0, 24.0, size=(n, 3)).astype(np.float32)
    v = np.zeros((n, 3), np.float32)
    v[:, 0] = vx
    return dict(x=(X / np.float32(32)).astype(np.float32), v=v, F=np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (n, 1)),
                b=np.zeros((n, 9), np.float32), mass=np.full(n, 6e-6, np.float32), vol=np.full(n, 1.5e-8, np.float32),
                ps=np.ones(n, np.float32), group=np.zeros(n, np.int32), id=np.arange(n, dtype=np.int64))


def test_error_codes():
    nb = (C.c_int32 * 3)(16, 16, 8)
    shape = (16, 16, 8)
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4)
    e.set_material(0, capi.MAT_SNOW, scenes.material_params(scenes.MAT_SNOW))
    L, h = e.L, e.h
    lo, hi, n = C.c_int32(0), C.c_int32(0), C.c_int64(0)
    f = C.c_float

    def schedule(t=0, max_units=64, lo_=C.byref(lo), hi_=C.byref(hi)):
        return L.mpmb_async_schedule(h, C.c_int64(t), f(1.0), f(0.1), f(1.0 / 32), f(4e4), C.c_int64(max_units), lo_, hi_)

    def advance(t=0, limit=1, dt=1e-4, n_=C.byref(n)):
        return L.mpmb_async_advance_level(h, C.c_int64(t), C.c_int32(limit), f(dt), n_)
    # before mpmb_async_init: MPMB_ERR_STATE (-4)
    assert schedule() == -4 and advance() == -4 and L.mpmb_async_block_state(h, None, None, None, None) == -4
    e.async_init(shape, 32.0)
    # bad arguments: MPMB_ERR_INVALID (-1)
    assert schedule(lo_=None) == -1 and schedule(hi_=None) == -1 and schedule(t=-1) == -1
    assert schedule(max_units=0) == -1 and schedule(max_units=(1 << 30) + 1) == -1
    for limit in (0, -2, 3, 6, 96, -(1 << 31)):
        assert advance(limit=limit) == -1, limit
    assert advance(t=-1) == -1 and advance(n_=None) == -1 and advance(dt=0.0) == -1 and advance(dt=float("inf")) == -1
    assert L.mpmb_async_block_state(h, None, None, None, None) == 0
    assert schedule(max_units=1 << 30) == 0 and (lo.value, hi.value) == (1, 1)       # no particles: every block at level 1
    assert advance(limit=1 << 30) == 0 and n.value == 0
    # a NaN velocity in a due block (every block is due at t = 0): MPMB_ERR_LIMIT (-5), the block state unchanged
    rng = np.random.default_rng(5)
    rec = _records(rng, 64)
    e.async_add(0, rec)
    assert schedule() == 0 and 1 <= lo.value <= hi.value <= 64
    assert advance(limit=lo.value) == 0 and n.value > 0
    before = e.async_block_state()
    assert (before["level"] > 1).any() and (before["particle_t"] > 0).any()
    e.async_add(0, dict(_records(rng, 1, vx=float("nan")), id=np.array([100])))
    assert schedule() == -5
    _same_state(before, e.async_block_state())
    # jelly in the pool while a block is due: MPMB_ERR_INVALID
    e.set_material(1, capi.MAT_JELLY, scenes.material_params(scenes.MAT_JELLY))
    e.async_init((16, 16, 8), 32.0)
    e.async_add(0, dict(rec, group=np.ones(64, np.int32)))
    assert schedule() == -1
    _same_state(e.async_block_state(), dict(level=np.ones(shape, np.int64), local_min=np.ones(shape, np.int64), particle_t=np.zeros(shape, np.int64),
                                            backup_t=np.zeros(shape, np.int64)))
    e.close()
    # z-slab ranks and rigid samples: MPMB_ERR_STATE
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4, world=2, rank=0, tile_z0=0, tile_z1=4, migrate_capacity=1024)
    L, h = e.L, e.h
    assert schedule() == -4 and advance() == -4 and L.mpmb_async_block_state(h, None, None, None, None) == -4
    e.close()
    e = _Engine((32, 32, 32), 1.0 / 32, 1e-4)
    L, h = e.L, e.h
    assert L.mpmb_async_init(h, nb, f(32.0)) == 0
    off, tri, rid = np.zeros(3, np.float32), np.zeros(9, np.float32), np.ones(1, np.int32)
    tri[3], tri[7] = 1.0, 1.0
    assert L.mpmb_set_rigid_samples(h, 2, C.c_int64(1), off.ctypes.data_as(C.c_void_p), tri.ctypes.data_as(C.c_void_p),
                                    rid.ctypes.data_as(C.c_void_p)) == 0
    assert schedule() == -4 and advance() == -4 and L.mpmb_async_block_state(h, None, None, None, None) == -4
    e.close()
