"""How AsyncMPM drives an engine that keeps the pools (mpmb_async_*): a stand-in engine records the mirror's calls and keeps
the pools with the host-pool code itself, running the substeps on the oracle.  Per scheduler iteration with a due block the
mirror makes one limits call, per level turn one advance whose flags are the host masks, and inside step() it never uploads
or downloads particles.  tests/test_gpu_async_device.py checks the device pools themselves."""
import numpy as np

from taichi_mpm_b200 import async_mpm, capi, scenes
from tests import common as T
from tests.test_async_host import OracleEngine

RES = (32, 32, 32)


class RecordingEngine(OracleEngine):
    """OracleEngine plus the mpmb_async_* calls, executed by a host-pool AsyncMPM (test infrastructure)."""

    def __init__(self, res, dx, dt, *a, **kw):
        super().__init__(res, dx, dt, *a, **kw)
        self.dx = dx
        self.calls = []
        self.shadow = None

    def upload(self, *a, **kw):
        self.calls.append(("upload",))
        return super().upload(*a, **kw)

    def download(self):
        self.calls.append(("download",))
        return super().download()

    def async_init(self, nb, inv_dx):
        self.calls.append(("init", tuple(nb), float(inv_dx)))
        inner = OracleEngine(self.scene["res"], self.dx, self.scene["dt"])
        inner.scene = self.scene                                    # the materials and the step the mirror sets
        sh = async_mpm.AsyncMPM.__new__(async_mpm.AsyncMPM)
        sh.nb, sh.delta_x, sh.engine = tuple(nb), self.dx, inner
        gx, gy, gz = np.meshgrid(*(np.arange(n) for n in sh.nb), indexing="ij")
        sh._offset = async_mpm._morton(gx, gy, gz)
        sh._on_device = False
        sh.pool = sh.backup = None
        self.shadow = sh

    def async_add(self, which, rec):
        self.calls.append(("add", which, len(rec["x"])))
        sh = self.shadow
        r = {k: np.asarray(rec[k]).copy() for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group", "id")}
        r["block"] = sh._block_of(r["x"])
        if which == 0:
            sh.pool = sh._cat(sh.pool, r)
        else:
            sh.backup = sh._cat(sh.backup, r)
        if sh.backup is None:
            sh.backup = sh._empty_like(r)

    def async_block_limits(self, with_limits):
        self.calls.append(("limits", bool(with_limits)))
        sh = self.shadow
        sh._groups = list(zip(self.scene["mat_kind"], self.scene["mat_params"]))
        nonempty, limits = sh._pool_scan(0)
        blk = np.flatnonzero(nonempty.reshape(-1)).astype(np.int32)
        if not with_limits:
            return blk, None, None
        try:
            mn, mx = limits()
        except ValueError as e:
            raise capi.MpmbError(-1, str(e))
        return blk, mn[blk], mx[blk]

    def async_advance(self, flags, dt):
        self.calls.append(("advance", np.asarray(flags, np.uint8).reshape(-1).copy(), float(dt)))
        fl = np.asarray(flags, np.uint8).reshape(self.shadow.nb)
        masks = [(fl & bit) != 0 for bit in (capi.ASYNC_SMALLER, capi.ASYNC_EQUAL, capi.ASYNC_LARGER, capi.ASYNC_SWAP, capi.ASYNC_CLEAR)]
        return self.shadow._advance_host(*masks, dt)

    def async_size(self):
        return tuple(0 if p is None else len(p["id"]) for p in (self.shadow.pool, self.shadow.backup))

    def async_download(self, which, fields=("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group")):
        sh = self.shadow
        p = (sh.pool, sh.backup)[which]
        b = p["block"]
        d = dict(p, id=p["id"].astype(np.uint32), block=((b[:, 0] * sh.nb[1] + b[:, 1]) * sh.nb[2] + b[:, 2]).astype(np.int32))
        return {k: d[k] for k in fields}


def _pair(monkeypatch):
    scene, st = T.perturbed_scene(scenes.MAT_SNOW, res=32, cells=8, seed=7, strain=0.0, vel=0.0, with_floor=False)
    st["v"][:] = 0
    st["v"][st["x"][:, 0] > 0.55, 0] = 10.0
    unit = 2.5e-5
    ms = []
    for cls in (OracleEngine, RecordingEngine):
        monkeypatch.setattr(capi, "Engine", cls)
        m = async_mpm.AsyncMPM(res=RES, base_delta_t=unit, unit_delta_t=unit, max_units=64, cfl_dt_mul=0.1, gravity=scene["gravity"])
        m.add_particles(type="snow", positions=st["x"], density=400.0)
        for k in ("v", "mass", "vol", "F", "b", "ps"):
            m.pool[k][:] = st[k]
        ms.append(m)
    return unit, ms[0], ms[1]


def test_mirror_makes_one_limits_call_per_due_iteration_and_one_advance_per_level_turn(monkeypatch):
    unit, mh, md = _pair(monkeypatch)
    assert not mh._device_pools and md._device_pools
    expected, due_iterations, iterations = [], [0], [0]

    real_advance_host = mh._advance_host

    def advance_host(smaller, equal, larger, swap, clear_b, dt):
        expected.append(((smaller * capi.ASYNC_SMALLER | equal * capi.ASYNC_EQUAL | larger * capi.ASYNC_LARGER | swap * capi.ASYNC_SWAP |
                          clear_b * capi.ASYNC_CLEAR).astype(np.uint8).reshape(-1), dt))
        return real_advance_host(smaller, equal, larger, swap, clear_b, dt)
    mh._advance_host = advance_host
    real_scan = mh._pool_scan

    def pool_scan(t):
        nonempty, limits = real_scan(t)

        def counted():
            due_iterations[0] += 1
            return limits()
        return nonempty, counted
    mh._pool_scan = pool_scan
    real_update = md.update_dt_limits

    def update():
        iterations[0] += 1
        return real_update()
    md.update_dt_limits = update

    for _ in range(2):
        mh.step(80 * unit)
        md.step(80 * unit)
        assert mh.scheduler_stats() == md.scheduler_stats()
    calls = md.engine.calls
    kinds = [c[0] for c in calls]
    assert kinds[0] == "init" and kinds[1] == "add" and "upload" not in kinds and "download" not in kinds
    assert calls[0][1] == md.nb and calls[0][2] == np.float32(32.0)
    limits = [c for c in calls if c[0] == "limits"]
    assert len(limits) == iterations[0] > 0                          # one pass over the pool per scheduler iteration
    assert sum(1 for c in limits if c[1]) == due_iterations[0] > 0     # with limits exactly when a block is due
    adv = [c for c in calls if c[0] == "advance"]
    assert len(adv) == len(expected) > 0
    for (_, fl, dt), (efl, edt) in zip(adv, expected):
        assert np.array_equal(fl, efl) and dt == edt
    for a, b in zip(mh.pools(), md.pools()):
        for k in ("id", "x", "v", "F"):
            assert np.array_equal(a[k], b[k])


def test_particles_added_after_the_first_step_go_to_the_engine_pool(monkeypatch):
    unit, mh, md = _pair(monkeypatch)
    md.step(40 * unit)
    n = md.num_particles()
    md.add_particles(type="snow", benchmark_block=((20, 20, 12), (22, 22, 14)))
    adds = [c for c in md.engine.calls if c[0] == "add"]
    assert adds[-1] == ("add", 0, 64) and md.pool is None and md.num_particles() == n + 64
    assert md.get_particles()["id"].max() == n + 63 and md.engine.shadow.pool["id"][-64:].tolist() == list(range(4096, 4160))
