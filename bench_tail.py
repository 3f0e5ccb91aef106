#!/usr/bin/env python
"""bench_tail.py — how long the CTAs of k_p2g and k_g2p sit idle while the slowest CTA of a launch finishes.

    python -m taichi_mpm_b200.build --define MPMB_TILE_TRACE --out build_variants/libmpmb_tile_trace.so
    python bench_tail.py [--lib build_variants/libmpmb_tile_trace.so] [--substeps 10] [--out FILE]

Runs bench.py's flagship scene (sand256, seeded on the device the same way) on one GPU with a library built with
-DMPMB_TILE_TRACE, where every CTA of the two tile kernels records its start and end (%globaltimer), its SM and the
tiles and particle rows it processed.  Two states, as bench.py times them: the column at rest (after the 20 warm-up
substeps) and the developed collapse (after the 20 + 2 * 200 + 20000 + 20 substeps that precede bench.py's flowing
timed region).  In each state `--substeps` single substeps are traced and, per kernel, averaged:

  span       first CTA start to last CTA end, us
  busy       mean and max CTA busy time (end - start), us
  idle       1 - sum(busy) / (span * CTAs): the share of the launch's CTA slots that wait for the slowest CTA;
             per SM the same over the CTAs that ran there (min / mean / max over the SMs)
  tiles, rows  per CTA (mean / min / max)
"""
import argparse
import ctypes as C
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KERNELS = ("k_p2g", "k_g2p")  # index = the `which` of mpmb_debug_tile_trace
TRACE = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("sm", "<i4"), ("tiles", "<i4"), ("rows", "<i4"), ("pad", "<i4")])


def read_trace(eng, which, cap=4096):
    buf = np.zeros(cap, TRACE)
    n = eng.L.mpmb_debug_tile_trace(eng.h, which, buf.ctypes.data_as(C.c_void_p), cap)
    if n < 0:
        raise RuntimeError("mpmb_debug_tile_trace failed: %d" % n)
    return buf[:min(n, cap)]


def launch_stats(t):
    t0, t1 = t["t0"].astype(np.int64), t["t1"].astype(np.int64)
    span = float(t1.max() - t0.min())
    busy = (t1 - t0).astype(np.float64)
    sm_idle = []
    for s in np.unique(t["sm"]):
        b = busy[t["sm"] == s]
        sm_idle.append(1.0 - b.sum() / (span * len(b)))
    return dict(span=span, busy_mean=float(busy.mean()), busy_max=float(busy.max()), idle=1.0 - busy.sum() / (span * len(busy)),
                sm_idle=np.array(sm_idle), tiles=t["tiles"].astype(np.float64), rows=t["rows"].astype(np.float64), ctas=len(t))


def summarize(samples):
    us = 1e-3
    s = {"ctas": samples[0]["ctas"],
         "span_us": float(np.mean([x["span"] for x in samples])) * us,
         "busy_mean_us": float(np.mean([x["busy_mean"] for x in samples])) * us,
         "busy_max_us": float(np.mean([x["busy_max"] for x in samples])) * us,
         "idle": float(np.mean([x["idle"] for x in samples])),
         "sm_idle": {k: float(np.mean([f(x["sm_idle"]) for x in samples])) for k, f in (("min", np.min), ("mean", np.mean), ("max", np.max))}}
    for key in ("tiles", "rows"):
        s[key + "_per_cta"] = {k: float(np.mean([f(x[key]) for x in samples])) for k, f in (("mean", np.mean), ("min", np.min), ("max", np.max))}
    return s


def trace_state(job, substeps):
    per = {k: [] for k in KERNELS}
    for _ in range(substeps):
        job.substep(1)
        for i, k in enumerate(KERNELS):
            per[k].append(launch_stats(read_trace(job.eng, i)))
    return {k: summarize(v) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "build_variants", "libmpmb_tile_trace.so"))
    ap.add_argument("--substeps", type=int, default=10, help="traced substeps per state")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--develop", type=int, default=20000)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not os.path.exists(args.lib):
        sys.exit("%s is missing: build it with python -m taichi_mpm_b200.build --define MPMB_TILE_TRACE --out %s" % (args.lib, args.lib))
    os.environ["MPMB_LIB"] = args.lib
    import torch
    import bench
    from taichi_mpm_b200 import capi
    L = capi.lib()
    L.mpmb_debug_tile_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    torch.cuda.set_device(0)
    cfg = bench.build_workload("sand256", 1.0, state=False)
    job = bench.SlabJob(types.SimpleNamespace(), cfg, 0, 1, 0, None)
    res = {"lib": os.path.basename(args.lib), "gpu": torch.cuda.get_device_name(0), "particles": job.n_total, "traced_substeps": args.substeps}
    clk = bench.ClockSampler(0)
    res["power_limit_w"], res["sm_max_mhz"] = clk.power_limit_w, clk.max_mhz
    job.substep(args.warmup)
    res["at_rest"] = trace_state(job, args.substeps)
    # bench.py's flowing timed region starts after its quiescent pass (warm-up, timed and profiled substeps), the develop
    # run and a second warm-up
    flowing_start = args.warmup + 2 * args.steps + args.develop + args.warmup
    job.substep(flowing_start - args.warmup - args.substeps)
    res["collapse"] = trace_state(job, args.substeps)
    job.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
