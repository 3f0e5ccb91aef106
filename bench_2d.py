"""Throughput of the 2-D engine (MPM<2>, MpmbConfig.dim = 2): a Drucker-Prager sand column on a floor plane (friction 0.4,
separating), 4 particles per cell, in million particle-updates per second (particles x substeps / wall time).

    python bench_2d.py [--steps K] [--warmup W] [--sizes 1024,2048] [--develop-time T] [--no-cpu-baseline]

Two sizes: a 1024^2 grid with a 512 x 512-cell column (1.05 M particles, dt = 5e-6) and a 2048^2 grid with a
1024 x 1024-cell column (4.19 M particles, dt = 2.5e-6); both are dt ~ dx / (5.7 c_P) for the sand's P-wave speed, the
margin of bench.py's sand collapse.  Each size is timed at rest (the column as seeded) and in a developed collapse (after
--develop-time seconds of simulated time), each with its per-stage times from the engine's CUDA events (a separate, profiled
window: profiling launches every kernel from the host).  The CPU baselines are one substep of the fp32 2-D oracle
(oracle/mpm_oracle.cpp, OpenMP in its grid update and G2P) on the same column and, where `build()` compiled the reference in place
(oracle/_ref/libtransfer2d_ref.so), one substep of the reference's own MPM<2>::substep() with every host thread.  The card's name
and power limit are read in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from taichi_mpm_b200 import capi, scenes  # noqa: E402

SIZES = {1024: (512, 5e-6), 2048: (1024, 2.5e-6)}
FLOOR = 8   # cells


def card(device):
    """Name, power limit and max SM clock of the card (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:   # the figures are still measured; the card is then unknown and says so
        return {"name": None, "power_limit_w": None, "error": repr(e)}


def column(res):
    cells, dt = SIZES[res]
    lo = ((res - cells) // 2, FLOOR)
    x, mass, vol = scenes.lattice_block2d((res, res), lo, (lo[0] + cells, lo[1] + cells), density=400.0)
    st = scenes.make_state2d(x, mass, vol, scenes.MAT_SAND)
    return st, dt


def p_wave_margin(res, dt):
    """dx / (c_P dt) of the sand at rest: c_P = sqrt((lambda + 2 mu) / rho)."""
    p = scenes.material_params(scenes.MAT_SAND)
    c = math.sqrt((p[1] + 2 * p[0]) / 400.0)
    return (1.0 / res) / (c * dt)


def engine_for(res, st, dt, device):
    e = capi.Engine2D((res, res), 1.0 / res, dt, (0.0, -10.0), device=device)
    e.set_material(0, scenes.MAT_SAND, scenes.material_params(scenes.MAT_SAND))
    e.set_planes([[0.0, 1.0, 0.0, -float(FLOOR)]], 0.4)
    e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    return e


def timed(e, steps, warmup, stage_steps):
    """Rate over `steps` replayed substeps (after `warmup`), then a profiled window of `stage_steps` for the stage times."""
    e.substep(warmup)
    e.synchronize()
    n0, u0 = e.num_particles(), e.update_count()
    t0 = time.perf_counter()
    e.substep(steps)
    e.synchronize()
    wall = time.perf_counter() - t0
    updates = e.update_count() - u0
    e.set_profiling(True)
    e.get_profile(reset=True)
    e.substep(stage_steps)
    ms, launches = e.get_profile(reset=True)
    e.set_profiling(False)
    names = ("ordering", "p2g_and_grid", "g2p")
    return {"particles": n0, "substeps": steps, "wall_s": wall, "mupdates_per_s": updates / wall / 1e6,
            "ms_per_substep": 1e3 * wall / steps,
            "stage_ms_per_substep": {k: ms[i] / stage_steps for i, k in enumerate(names)},
            "stage_launches_per_substep": {k: launches[i] / stage_steps for i, k in enumerate(names)}}


def cpu_baseline(st, res, dt, reps):
    """Seconds per substep of the fp32 2-D oracle on the same column, best of `reps`."""
    from oracle import pyoracle2d as O
    scene = dict(res=(res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0), particle_gravity=1, clean_boundary=1,
                 mat_kind=np.array([scenes.MAT_SAND], np.int32), mat_params=scenes.material_params(scenes.MAT_SAND)[None],
                 sdf=scenes.planes_sdf2d((res, res), [[0.0, 1.0, 0.0, -float(FLOOR)]]), friction=0.4)
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        O.substep2d(scene, st, np.float32, want_grids=False)
        best = min(best, time.perf_counter() - t0)
    return {"impl": "fp32 2-D oracle (serial P2G; OpenMP grid update and G2P)", "threads": int(O.lib().oracle_fast_num_threads()), "s_per_substep": best,
            "mupdates_per_s": len(st["x"]) / best / 1e6}


def cpu_reference(st, res, dt):
    """Seconds per substep of the reference's MPM<2>::substep() compiled in place, on the same column (None where it was not
    built: this benchmark compiles nothing)."""
    from oracle import pyoracle2d as O
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libtransfer2d_ref.so")):
        return None
    scene = dict(res=(res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0), particle_gravity=1, clean_boundary=1,
                 mat_kind=np.array([scenes.MAT_SAND], np.int32), mat_params=scenes.material_params(scenes.MAT_SAND)[None],
                 planes=np.array([[0.0, 1.0, 0.0, -float(FLOOR)]], np.float32), friction=0.4)
    r = O.RefSolver2D(scene, st)
    threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    r.set_threads(threads)
    r.substep(1)   # first touch of the grid pages
    t0 = time.perf_counter()
    r.substep(1)
    s = time.perf_counter() - t0
    r.close()
    return {"impl": "the reference's MPM<2>::substep() compiled in place", "threads": threads, "s_per_substep": s,
            "mupdates_per_s": len(st["x"]) / s / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--stage-steps", type=int, default=20)
    ap.add_argument("--sizes", default="1024,2048")
    ap.add_argument("--develop-time", type=float, default=0.05, help="simulated seconds before the developed-collapse measurement")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--cpu-reps", type=int, default=2)
    args = ap.parse_args()
    line = {"metric": "mpm2d_sand_column_mupdates_per_s", "unit": "M particle-updates/s", "card": card(args.device), "sizes": []}
    for res in (int(s) for s in args.sizes.split(",")):
        st, dt = column(res)
        e = engine_for(res, st, dt, args.device)
        entry = {"res": [res, res], "column_cells": SIZES[res][0], "dt": dt, "dx_over_cP_dt": p_wave_margin(res, dt)}
        entry["at_rest"] = timed(e, args.steps, args.warmup, args.stage_steps)
        develop = int(round(args.develop_time / dt))
        e.substep(develop)
        entry["developed"] = dict(timed(e, args.steps, 0, args.stage_steps), develop_substeps=develop)
        if not args.no_cpu_baseline:
            entry["cpu_baseline"] = cpu_baseline(st, res, dt, args.cpu_reps)
            entry["speedup_vs_cpu_oracle"] = entry["developed"]["mupdates_per_s"] / entry["cpu_baseline"]["mupdates_per_s"]
        if not args.no_cpu_baseline:
            ref = cpu_reference(st, res, dt)
            entry["cpu_reference_mpm2"] = ref if ref is not None else "not available: oracle/_ref was not built"
            if ref is not None:
                entry["speedup_vs_cpu_reference"] = entry["developed"]["mupdates_per_s"] / ref["mupdates_per_s"]
        e.close()
        line["sizes"].append(entry)
    line["value"] = line["sizes"][0]["developed"]["mupdates_per_s"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
