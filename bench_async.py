"""AsyncMPM on a 128^3 grid with 1.05 M snow particles, half of them moving at 10 m/s so that two time levels are active
(cfl_dt_mul = 0.1) — the scheduler's pools kept two ways, from the same seeded state:

  host     numpy record arrays: every advance gathers its set on the host, uploads it, runs the substep and downloads the
           survivors (what an engine without the mpmb_async_* calls gets)
  device   the engine's pools (mpmb_async_*): no particle record crosses the bus inside step()

    python bench_async.py [--steps 3] [--warmup 1]

Prints one JSON line: the card and its power limit (read in the same run) and, per leg, ms per AsyncMPM.step (wall time ending
in a device synchronise, over --steps steps after --warmup), advances and gathered particles per step and particle updates per
second.  Both legs must end with bitwise-equal pools.  Needs a CUDA device."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

UNIT = 1e-5
STEP_UNITS = 32   # one step = one period of the slow level


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    limit = None
    try:
        import pynvml
        pynvml.nvmlInit()
        limit = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    return name, limit


def model(host):
    from taichi_mpm_b200 import async_mpm, capi
    real = capi.Engine

    class HostPoolsEngine:
        """The engine without its mpmb_async_* calls: AsyncMPM keeps the pools on the host."""

        def __init__(self, *a, **kw):
            self._e = real(*a, **kw)

        def __getattr__(self, name):
            if name.startswith("async_"):
                raise AttributeError(name)
            return getattr(self._e, name)

    capi.Engine = HostPoolsEngine if host else real
    try:
        m = async_mpm.AsyncMPM(res=(128, 128, 128), base_delta_t=UNIT, unit_delta_t=UNIT, max_units=64, cfl_dt_mul=0.1)
    finally:
        capi.Engine = real
    m.add_particles(type="snow", benchmark_block=((32, 20, 32), (64, 52, 96)))
    m.add_particles(type="snow", benchmark_block=((64, 20, 32), (96, 52, 96)), initial_velocity=(10.0, 0.0, 0.0))
    assert m._device_pools == (not host)
    return m


def leg(host, steps, warmup):
    m = model(host)
    n = m.num_particles()
    advances = [0]
    real_advance = m.advance

    def counted(limit):
        advances[0] += 1
        return real_advance(limit)
    m.advance = counted
    for _ in range(warmup):
        m.step(STEP_UNITS * UNIT)
    m.engine.synchronize()
    a0, u0 = advances[0], m.update_counter
    t0 = time.perf_counter()
    for _ in range(steps):
        m.step(STEP_UNITS * UNIT)
    m.engine.synchronize()
    dt = time.perf_counter() - t0
    upd = m.update_counter - u0
    st = m.scheduler_stats()
    out = dict(ms_per_step=1e3 * dt / steps, advances_per_step=(advances[0] - a0) / steps, gathered_per_step=upd / steps,
               particle_updates_per_s=upd / dt, levels=[st["min_level"], st["max_level"]], particles=n)
    return out, m.pools()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_async.py needs a CUDA device")
    name, limit = card()
    res = {}
    pools = {}
    for which in ("device", "host"):
        res[which], pools[which] = leg(which == "host", a.steps, a.warmup)
    for ph, pd in zip(pools["host"], pools["device"]):
        assert len(ph["id"]) == len(pd["id"])
        for k in ("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group"):
            x, y = np.ascontiguousarray(ph[k]), np.ascontiguousarray(pd[k])
            assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y), k
    print(json.dumps(dict(bench="async_snow128", gpu=name, power_limit_w=limit, steps=a.steps, warmup=a.warmup, step_units=STEP_UNITS,
                          unit_delta_t=UNIT, legs=res, speedup=res["host"]["ms_per_step"] / res["device"]["ms_per_step"], pools_equal=True)))


if __name__ == "__main__":
    main()
