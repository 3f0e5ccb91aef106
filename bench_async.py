"""AsyncMPM on a 128^3 grid with 1.05 M snow particles, half of them moving at 10 m/s so that two time levels are active
(cfl_dt_mul = 0.1) — the scheduler's pools and block state kept three ways, from the same seeded state:

  host          numpy record arrays: every advance gathers its set on the host, uploads it, runs the substep and downloads
                the survivors (what an engine without the mpmb_async_* calls gets); the numpy scheduler
  device_pools  the engine's pools (mpmb_async_*): no particle record crosses the bus inside step(); the numpy scheduler
                (the engine's mpmb_async_schedule / mpmb_async_advance_level hidden)
  device        the engine's pools and its block scheduler: update_dt_limits and advance are one engine call each

    python bench_async.py [--steps 3] [--warmup 1]

Prints one JSON line: the card and its power limit (read in the same run) and, per leg and for each of two runs (the legs
alternate: host, device_pools, device, then the reverse), ms per AsyncMPM.step (wall time ending in a device synchronise, over
--steps steps after --warmup), ms per step spent inside update_dt_limits, advances and gathered particles per step and
particle updates per second.  All legs must end with bitwise-equal pools.  Needs a CUDA device."""
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


LEGS = ("host", "device_pools", "device")
HIDDEN = {"host": lambda name: name.startswith("async_"),
          "device_pools": lambda name: name in ("async_schedule", "async_advance_level", "async_block_state"),
          "device": lambda name: False}


def model(which):
    from taichi_mpm_b200 import async_mpm, capi
    real = capi.Engine
    hidden = HIDDEN[which]

    class HidingEngine:
        """The engine without some of its mpmb_async_* calls: AsyncMPM then does that part on the host."""

        def __init__(self, *a, **kw):
            self._e = real(*a, **kw)

        def __getattr__(self, name):
            if hidden(name):
                raise AttributeError(name)
            return getattr(self._e, name)

    capi.Engine = HidingEngine
    try:
        m = async_mpm.AsyncMPM(res=(128, 128, 128), base_delta_t=UNIT, unit_delta_t=UNIT, max_units=64, cfl_dt_mul=0.1)
    finally:
        capi.Engine = real
    m.add_particles(type="snow", benchmark_block=((32, 20, 32), (64, 52, 96)))
    m.add_particles(type="snow", benchmark_block=((64, 20, 32), (96, 52, 96)), initial_velocity=(10.0, 0.0, 0.0))
    assert (m._device_pools, m._device_sched) == {"host": (False, False), "device_pools": (True, False), "device": (True, True)}[which]
    return m


def leg(which, steps, warmup):
    m = model(which)
    n = m.num_particles()
    advances = [0]
    sched_s = [0.0]
    real_advance, real_update = m.advance, m.update_dt_limits

    def counted(limit):
        advances[0] += 1
        return real_advance(limit)

    def timed():
        t = time.perf_counter()
        real_update()
        sched_s[0] += time.perf_counter() - t
    m.advance, m.update_dt_limits = counted, timed
    for _ in range(warmup):
        m.step(STEP_UNITS * UNIT)
    m.engine.synchronize()
    a0, u0, s0 = advances[0], m.update_counter, sched_s[0]
    t0 = time.perf_counter()
    for _ in range(steps):
        m.step(STEP_UNITS * UNIT)
    m.engine.synchronize()
    dt = time.perf_counter() - t0
    upd = m.update_counter - u0
    st = m.scheduler_stats()
    out = dict(ms_per_step=1e3 * dt / steps, ms_update_dt_limits_per_step=1e3 * (sched_s[0] - s0) / steps,
               advances_per_step=(advances[0] - a0) / steps, gathered_per_step=upd / steps, particle_updates_per_s=upd / dt,
               levels=[st["min_level"], st["max_level"]], particles=n)
    pools = m.pools()
    m.engine.close()
    return out, pools


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_async.py needs a CUDA device")
    name, limit = card()
    res = {w: [] for w in LEGS}
    for order in (LEGS, LEGS[::-1]):
        ref = None
        for which in order:
            out, pools = leg(which, a.steps, a.warmup)
            res[which].append(out)
            if ref is None:
                ref = pools
                continue
            for pr, pw in zip(ref, pools):
                assert len(pr["id"]) == len(pw["id"]), which
                for k in ("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group"):
                    x, y = np.ascontiguousarray(pr[k]), np.ascontiguousarray(pw[k])
                    assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y), (which, k)
    best = {w: min(r["ms_per_step"] for r in res[w]) for w in LEGS}
    print(json.dumps(dict(bench="async_snow128", gpu=name, power_limit_w=limit, steps=a.steps, warmup=a.warmup, step_units=STEP_UNITS,
                          unit_delta_t=UNIT, legs=res, speedup_over_host=best["host"] / best["device"],
                          speedup_over_device_pools=best["device_pools"] / best["device"], pools_equal=True)))


if __name__ == "__main__":
    main()
