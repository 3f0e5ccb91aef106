"""The drop-in end to end on a pool that mixes particle types: BASELINE config 3's 8 M particles (256^3 grid, a 100^3-cell block,
dt = 2e-5, floor plane) in the reference's 320-byte slots in pinned host memory, each frame mpmb_upload_aos -> mpmb_substep(500)
-> mpmb_download_aos (INTEGRATION.md §2), in million particle-updates per second (survivors x substeps / wall time of the frame).

    python bench_dropin_mixed.py [--frames F] [--substeps S] [--scale X]

Two legs, run in the order single, mixed, mixed, single:
  single  the block as one sand pool, the single-offset layout (off_scalar = SandParticle::logJp), as bench.py's e2e leg;
  mixed   the block as four equal slabs along x of sand, snow, water and visco, one material group each, with the per-kind
          scalar offsets of MpmbAosLayout.off_scalar_by_kind.
The slot offsets are the values reft_aos_layout / reft_aos_scalar_offsets take by offsetof() on the reference's classes
(oracle/transfer_mixed_ref.cpp); the copied window is the byte range of every slot that crosses the bus in each direction.  A
warm frame precedes the timed ones.  The card's name and power limit are read in the same run.  Prints one JSON line; writes
nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from taichi_mpm_b200 import capi, scenes  # noqa: E402

SLOT = dict(stride=320, off_pos=32, off_v_and_m=16, off_dg_e=48, off_apic_b=96, col_pitch=16, off_vol=164)
SCALAR = {scenes.MAT_SNOW: 196, scenes.MAT_WATER: 204, scenes.MAT_SAND: 216, scenes.MAT_VISCO: 196}
MIXED = (scenes.MAT_SAND, scenes.MAT_SNOW, scenes.MAT_WATER, scenes.MAT_VISCO)


def card(device=0):
    """Name and power limit of the card (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:
        return {"name": None, "power_limit_w": None, "error": repr(e)}


def layout(mixed):
    L = capi.MpmbAosLayout()
    for k, v in SLOT.items():
        setattr(L, k, v)
    if mixed:
        L.set_scalar_offsets(SCALAR)
    else:
        L.off_scalar = SCALAR[scenes.MAT_SAND]
    return L


def window(L):
    """[lo, hi) of every slot that crosses the bus: the rule of aos_window in mpmb_engine.cu."""
    mat = 2 * L.col_pitch + 12
    a = min(L.off_pos, L.off_v_and_m, L.off_dg_e, L.off_apic_b, L.off_vol)
    b = max(L.off_pos + 12, L.off_v_and_m + 16, L.off_dg_e + mat, L.off_apic_b + mat, L.off_vol + 4)
    offs = [L.off_scalar] + [o for o in L.off_scalar_by_kind if o > 0]
    for o in offs:
        if o >= 0:
            a, b = min(a, o), max(b, o + 4)
    return max(0, a & ~15), min(L.stride, (b + 15) & ~15)


def fill(pool, st, L, kinds):
    """The particles into slots 0..n-1 (id order), each type's scalar at its offset."""
    n = len(st["x"])
    f = pool.view(np.float32).reshape(-1, L.stride // 4)[:n]
    f[:, L.off_pos // 4: L.off_pos // 4 + 3] = st["x"]
    f[:, L.off_v_and_m // 4: L.off_v_and_m // 4 + 3] = st["v"]
    f[:, L.off_v_and_m // 4 + 3] = st["mass"]
    for c in range(3):
        o = (L.off_dg_e + c * L.col_pitch) // 4
        f[:, o: o + 3] = st["F"][:, 3 * c: 3 * c + 3]
        o = (L.off_apic_b + c * L.col_pitch) // 4
        f[:, o: o + 3] = st["b"][:, 3 * c: 3 * c + 3]
    f[:, L.off_vol // 4] = st["vol"]
    kind_of = np.asarray(kinds)[st["group"]]
    for k in set(kinds):
        off = SCALAR[k] if L.off_scalar == -1 else L.off_scalar
        f[kind_of == k, off // 4] = scenes.default_scalar(k)


def run_leg(cfg, mixed, pool_t, idx_t, frames, substeps):
    scene, st = cfg["scene"], cfg["state"]
    n, res = len(st["x"]), scene["res"]
    kinds = list(MIXED) if mixed else [scenes.MAT_SAND]
    st = dict(st)
    lo, hi = cfg["meta"]["lo"][0], cfg["meta"]["hi"][0]
    cell = np.floor(st["x"][:, 0] * res[0]).astype(np.int64)
    st["group"] = (np.clip((cell - lo) * len(kinds) // (hi - lo), 0, len(kinds) - 1) if mixed else np.zeros(n)).astype(np.int32)
    L = layout(mixed)
    pool, idx = pool_t.numpy(), idx_t.numpy().view(np.uint32)
    fill(pool, st, L, kinds)
    e = capi.Engine(res, scene["dx"], scene["dt"], gravity=scene["gravity"])
    try:
        for g, k in enumerate(kinds):
            e.set_material(g, k, scenes.material_params(k))
        e.set_planes(scene["planes"], scene["friction"])
        grp = st["group"]
        alive, times = n, []
        idx[:] = np.arange(n, dtype=np.uint32)
        for f in range(frames + 1):
            t0 = time.perf_counter()
            e.upload_aos(pool, idx[:alive], L, group=grp[idx[:alive]])
            e.substep(substeps)
            alive = e.download_aos(pool, idx[:alive], L)
            if f > 0:   # frame 0 warms the staging buffers and captures the graphs
                times.append(time.perf_counter() - t0)
        sec = float(np.median(times))
        w = window(L)
        return dict(leg="mixed" if mixed else "single", kinds=[int(k) for k in kinds], particles=n, alive=int(alive),
                    updates_per_s_M=alive * substeps / sec / 1e6, frame_seconds=sec, frame_seconds_all=[float(t) for t in times],
                    window=list(w), window_bytes_per_slot=w[1] - w[0], copied_bytes_each_way=(w[1] - w[0]) * n)
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--substeps", type=int, default=500)
    ap.add_argument("--scale", type=float, default=1.0, help="shrinks grid and block (config 3 at 1.0)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropin_mixed.py measures on a CUDA device; none is visible")
    cfg = scenes.config("sand256", scale=args.scale)
    n = len(cfg["state"]["x"])
    pool_t = torch.zeros(n * SLOT["stride"], dtype=torch.uint8, pin_memory=True)
    idx_t = torch.empty(n, dtype=torch.int32, pin_memory=True)
    legs = [run_leg(cfg, m, pool_t, idx_t, args.frames, args.substeps) for m in (False, True, True, False)]
    print(json.dumps(dict(workload="sand256 x%g drop-in, single vs mixed pool" % args.scale, substeps_per_frame=args.substeps,
                          frames=args.frames, card=card(), legs=legs)))


if __name__ == "__main__":
    main()
