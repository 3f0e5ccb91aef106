"""Rigid-coupled substeps on BASELINE config 2 (128^3 grid, 1.0 M jelly particles) with a scripted paddle, a free box and a floor
plane with the rigid-body level-set collision on — three ways of advancing the bodies, from the same start:

  host       the per-substep C-ABI contract with host advection: set_rigid_state -> substep(1) -> get_rigid_state -> level-set
             collision + HostRigidBody.advect in numpy (boundary samples uploaded once: the fair form of that contract)
  device     mpmb_set_rigid_motion: one script table + mpmb_substep(h, frame) per frame, CUDA graphs replayed
  no_graph   the same with no_graph=1 (every kernel launched from the host)

    python bench_rigid.py [--steps 200] [--warmup 20] [--frame 50]

Prints one JSON line: the card and its power limit (read in the same run), ms per substep of each leg (wall time ending in a
device synchronise, over --steps substeps after --warmup), and the differences of the legs' end states against the host leg
(body positions and velocities, particle centre of mass and momentum).  Needs a CUDA device."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


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


def scene(res, no_graph=False):
    from taichi_mpm_b200 import capi, mpm as mpm_mod, scenes
    m = mpm_mod.MPM(res=(res, res, res), base_delta_t=1e-4, gravity=(0.0, -10.0, 0.0), penalty=1e3, rigid_body_levelset_collision=True)
    if no_graph:
        m.engine.close()
        m.engine = capi.Engine(m.res, m.delta_x, m.base_delta_t, m.gravity, True, True, no_graph=True)
    ls = m.create_levelset()
    ls.add_plane((0, 1, 0), -20.0 / res)
    ls.set_friction(0.4)
    m.set_levelset(ls, False)
    lo = (res - 50) // 2
    m.add_particles(type="jelly", benchmark_block=((lo, 20, lo), (lo + 50, 70, lo + 50)), density=400.0, jitter=0.2, E=2e4)   # 1.0 M
    c = (lo + 25) / res
    m.add_particles(type="rigid", tris=scenes.plate_mesh(0.02, 0.15, axis=0), codimensional=True, friction=0.3,
                    scripted_position=lambda t: (c - 0.12 + 0.8 * t, 45.0 / res, c), scripted_rotation=lambda t: (0.0, 200.0 * t, 10.0))
    m.add_particles(type="rigid", tris=scenes.box_mesh((0.04, 0.03, 0.04)), codimensional=False, density=400.0, friction=0.3,
                    initial_position=(c + 0.1, 72.0 / res + 0.04, c + 0.05), initial_velocity=(-0.3, -1.0, 0.0), initial_rotation=(10.0, 20.0, 5.0))
    m._push()
    return m


def host_leg(m, n):
    """The per-substep contract: state in, one substep, velocities out, level-set collision and advect on the host."""
    from taichi_mpm_b200 import rigid as rigid_mod
    h = np.float32(m.base_delta_t)
    t = np.float32(m.current_t)
    if m._rigid_dirty:
        rec = m._rigid_records()
        m.engine.set_rigid(rec)
        m._samples = rec
        m._rigid_dirty = False
    rec = m._samples
    ls = m._levelset
    phi = ls.node_phi()
    ls.node_phi = lambda: phi      # the level set is static: its node values once, not per sample call
    for _ in range(n):
        m.engine.set_rigid_state(rigid_mod.state_records(m.rigids))
        m.engine.substep(1)
        rs = m.engine.get_rigid_state(len(m.rigids) + 1)
        for k, b in enumerate(m.rigids):
            b.velocity = rs["velocity"][k + 1].astype(np.float64)
            b.angular_velocity = rs["angular_velocity"][k + 1].astype(np.float64)
            sel = rec["sample_rigid"] == k + 1
            world = b.position + rec["sample_offset"][sel].astype(np.float64) @ b.rotation.T
            X = world / m.delta_x
            grad = np.stack([(ls.sample(X + e) - ls.sample(X - e)) / 0.5 for e in np.eye(3) * 0.25], 1)
            b.levelset_collision(world, ls.sample(X), grad / np.maximum(np.linalg.norm(grad, axis=1, keepdims=True), 1e-12))
        for b in m.rigids:
            b.advect(float(t), float(h), m.gravity)
        t = np.float32(t + h)
    m.current_t = t


def device_leg(m, n, frame):
    done = 0
    while done < n:
        k = min(frame, n - done)
        m.current_t = m._rigid_substeps(k)
        done += k


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def end_state(m):
    p = m.engine.download()
    mass = p["mass"].astype(np.float64)[:, None]
    return dict(bodies=[(b.position.copy(), b.velocity.copy()) for b in m.rigids], com=(mass * p["x"]).sum(0) / mass.sum(),
                momentum=(mass * p["v"]).sum(0), n=len(p["x"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--frame", type=int, default=50)
    ap.add_argument("--res", type=int, default=128)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_rigid.py needs a CUDA device")
    name, limit = card()
    legs = {"host": scene(a.res), "device": scene(a.res), "no_graph": scene(a.res, no_graph=True)}
    run = {"host": lambda m, n: host_leg(m, n), "device": lambda m, n: device_leg(m, n, a.frame), "no_graph": lambda m, n: device_leg(m, n, a.frame)}
    ms = {}
    for k, m in legs.items():
        run[k](m, a.warmup)
        ms[k] = timed(lambda: run[k](m, a.steps)) / a.steps
    ends = {k: end_state(m) for k, m in legs.items()}
    ref = ends["host"]
    diff = {}
    for k in ("device", "no_graph"):
        e = ends[k]
        diff[k] = dict(body_position=max(float(np.abs(p - q).max()) for (p, _), (q, _) in zip(e["bodies"], ref["bodies"])),
                       body_velocity=max(float(np.abs(v - w).max() / max(np.abs(w).max(), 1e-30)) for (_, v), (_, w) in zip(e["bodies"], ref["bodies"])),
                       com=float(np.abs(e["com"] - ref["com"]).max()),
                       momentum_rel=float(np.abs(e["momentum"] - ref["momentum"]).max() / max(np.abs(ref["momentum"]).max(), 1e-30)),
                       same_count=e["n"] == ref["n"])
    print(json.dumps(dict(bench="rigid_config2", card=name, power_limit_w=limit, particles=ref["n"], res=a.res, steps=a.steps, warmup=a.warmup,
                          frame=a.frame, ms_per_substep={k: round(v, 4) for k, v in ms.items()},
                          speedup_vs_host={k: round(ms["host"] / ms[k], 2) for k in ("device", "no_graph")},
                          end_state_diff_vs_host=diff)))


if __name__ == "__main__":
    main()
