"""Edits of the resident set on the flagship workload (sand256: 8 M sand particles, 256^3): the device edits
(mpmb_append_particles, mpmb_delete_inside_levelset) against the former host round trip (download -> concatenate or
filter -> upload), on two engines in the same state.

    python bench_resident_edit.py [--warmup 20]

Prints one JSON line: the card and its power limit (read in the same run), the wall time of each edit with a device
synchronise, the first substep after the edit against a steady one (device events, mpmb_get_profile), and whether both
paths leave the same live set (matched by position: the round trip renumbers the particles).  Needs a CUDA device: on a
machine without one it exits with an error instead of measuring anything else."""
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


def engine(cfg, warmup):
    from taichi_mpm_b200 import capi
    sc, m = cfg["scene"], cfg["meta"]
    e = capi.Engine(sc["res"], sc["dx"], sc["dt"], sc["gravity"], sc["particle_gravity"], True)
    e.set_material(0, m["kind"], sc["mat_params"][0])
    e.set_planes(sc["planes"], sc["friction"])
    e.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
    e.substep(warmup)
    e.synchronize()
    return e


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def substep_ms(e):
    """(first substep after the edit, the next one): device time summed over the stages (mpmb_get_profile)."""
    out = []
    e.set_profiling(True)
    for _ in range(2):
        e.get_profile(reset=True)
        e.substep(1)
        ms, _ = e.get_profile(reset=True)
        out.append(sum(ms))
    e.set_profiling(False)
    return out


def same_live_set(a, b):
    """Both downloads hold the same particles: positions sorted lexicographically, compared field by field."""
    if len(a["x"]) != len(b["x"]):
        return False, None
    oa, ob = np.lexsort(a["x"].T[::-1]), np.lexsort(b["x"].T[::-1])
    dx = float(np.abs(a["x"][oa] - b["x"][ob]).max()) if len(oa) else 0.0
    same = dx == 0.0 and all(np.array_equal(a[k][oa], b[k][ob]) for k in ("v", "F", "b", "mass", "vol", "ps", "group"))
    return bool(same), dx


def round_trip(e, edit):
    """The former mirror path: every resident particle to the host, edited there, everything uploaded again."""
    d = e.download()
    h = edit({k: d[k] for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")})
    e.upload(h["x"], h["v"], h["mass"], h["vol"], h["F"], h["b"], h["ps"], h["group"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20, help="substeps before each edit")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_resident_edit.py needs a CUDA device (an H100); nothing was measured")
    from taichi_mpm_b200 import mpm as mpm_mod, scenes
    name, limit = card()
    cfg = scenes.config("sand256", 1.0, state=False)
    sc, m = cfg["scene"], cfg["meta"]
    res, dx = m["res"], sc["dx"]
    out = {"metric": "resident_set_edit", "workload": "sand256", "gpu": name, "power_limit_w": limit, "warmup_substeps": args.warmup}
    for label, layers in (("append_1pct", 1), ("append_10pct", 10)):
        # a slab of the 8-per-cell lattice above the column: 100 x layers x 100 cells = 80 000 particles per layer
        x, mass, vol = scenes.lattice_block(res, (m["lo"][0], 120, m["lo"][2]), (m["hi"][0], 120 + layers, m["hi"][2]), m["density"], dx=dx)
        st = scenes.make_state(x, mass, vol, m["kind"])
        new = {k: st[k] for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
        dev, old = engine(cfg, args.warmup), engine(cfg, args.warmup)
        n0 = dev.num_particles()
        first, t_dev = timed(lambda: dev.append(new["x"], new["v"], new["mass"], new["vol"], new["F"], new["b"], new["ps"], new["group"]))
        _, t_old = timed(lambda: round_trip(old, lambda h: {k: np.concatenate([h[k], new[k]]) for k in h}))
        same, dpos = same_live_set(dev.download(), old.download())
        s_dev, s_old = substep_ms(dev), substep_ms(old)
        out[label] = {"n_resident": n0, "n_new": len(new["x"]), "first_id": first, "device_ms": t_dev, "round_trip_ms": t_old,
                      "first_substep_ms": s_dev[0], "steady_substep_ms": s_dev[1], "round_trip_first_substep_ms": s_old[0],
                      "live_sets_equal": same, "max_position_diff": dpos}
        dev.close(); old.close()
    # delete: a plane through the middle of the column (phi < 0 below it)
    ycut = 0.5 * (m["lo"][1] + m["hi"][1])
    cut = np.array([[0.0, 1.0, 0.0, -ycut]], np.float32)
    ls = mpm_mod.LevelSet((res,) * 3, dx)
    ls.add_plane((0.0, 1.0, 0.0), -ycut * dx)
    dev, old = engine(cfg, args.warmup), engine(cfg, args.warmup)
    n0 = dev.num_particles()
    for e in (dev, old):
        e.set_planes(cut, sc["friction"])
    n_del, t_dev = timed(dev.delete_inside_levelset)

    def keep_outside(h):
        keep = ~(ls.sample(h["x"].astype(np.float64) / dx) < 0)
        return {k: np.ascontiguousarray(a[keep]) for k, a in h.items()}

    _, t_old = timed(lambda: round_trip(old, keep_outside))
    same, dpos = same_live_set(dev.download(), old.download())
    s_dev, s_old = substep_ms(dev), substep_ms(old)
    out["delete_plane"] = {"n_resident": n0, "n_deleted": n_del, "device_ms": t_dev, "round_trip_ms": t_old, "first_substep_ms": s_dev[0],
                           "steady_substep_ms": s_dev[1], "round_trip_first_substep_ms": s_old[0], "live_sets_equal": same,
                           "max_position_diff": dpos}
    dev.close(); old.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
