"""The 2-D drop-in end to end: bench_2d.py's sand column (1024^2 grid, 1.05 M particles; 2048^2, 4.19 M) in MPM<2>'s own pool
of 192-byte ParticleContainer<2> slots in pinned host memory, in million particle-updates per second (survivors x substeps /
wall time of the frame).

    python bench_dropin_2d.py [--frames F] [--substeps S] [--sizes 1024,2048]

Three legs per size, each the median of F frames after a warm one:
  aos        mpmb_upload_aos -> mpmb_substep(S) -> mpmb_download_aos (INTEGRATION.md §2 on a 2-D handle);
  fieldwise  what a patched MPM<2>::substep() had to do without it: gather the pool into arrays, mpmb_upload_particles,
             mpmb_substep(S), mpmb_download_particles, scatter back into the slots by id and compact the index vector;
  substeps   mpmb_substep(S) alone, on the resident particles.
The aos and fieldwise legs start from the same pool and must leave byte-identical pools and index vectors (checked).  Bytes
per direction are what crosses the bus per frame.  The slot offsets are those reft2_aos_layout takes by offsetof() on the
in-place reference build's classes (oracle/transfer2d_aos_ref.cpp), written here because that build is not where this runs.
The card's name and power limit are read in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import bench_2d as B  # noqa: E402
from taichi_mpm_b200 import capi, scenes  # noqa: E402

# ParticleContainer<2> of the in-place reference build; off_scalar = SandParticle<2>::logJp
SLOT = dict(stride=192, off_pos=32, off_v_and_m=16, off_dg_e=40, off_apic_b=56, col_pitch=8, off_vol=84, off_scalar=136)
FIELDWISE_UP = 4 * (2 + 2 + 4 + 4 + 1 + 1 + 1)    # x, v, F, b, mass, vol, scalar per particle
FIELDWISE_DOWN = 4 * (1 + 2 + 2 + 4 + 4 + 4)      # key, x, v, F, b, (mass, vol, scalar, tag) per stored row


def layout():
    L = capi.MpmbAosLayout()
    for k, v in SLOT.items():
        setattr(L, k, v)
    return L


def window(L):
    """[lo, hi) of every slot that crosses the bus: the rule of aos_window in mpmb_engine.cu for dim = 2."""
    mat = L.col_pitch + 8
    a = min(L.off_pos, L.off_v_and_m, L.off_dg_e, L.off_apic_b, L.off_vol, L.off_scalar)
    b = max(L.off_pos + 8, L.off_v_and_m + 12, L.off_dg_e + mat, L.off_apic_b + mat, L.off_vol + 4, L.off_scalar + 4)
    return max(0, a & ~15), min(L.stride, (b + 15) & ~15)


def columns(L):
    """float32 column indices of x, v, mass, F, b, vol, scalar in a slot."""
    o = lambda off, k: [off // 4 + i for i in range(k)]
    F = o(L.off_dg_e, 2) + o(L.off_dg_e + L.col_pitch, 2)
    b = o(L.off_apic_b, 2) + o(L.off_apic_b + L.col_pitch, 2)
    return dict(x=o(L.off_pos, 2), v=o(L.off_v_and_m, 2), mass=L.off_v_and_m // 4 + 2, F=F, b=b, vol=L.off_vol // 4, ps=L.off_scalar // 4)


def fill(pool, st, L):
    f = pool.view(np.float32).reshape(-1, L.stride // 4)
    for k, c in columns(L).items():
        f[: len(st["x"]), c] = st[k]


def engine(res, dt):
    e = capi.Engine2D((res, res), 1.0 / res, dt, (0.0, -10.0))
    e.set_material(0, scenes.MAT_SAND, scenes.material_params(scenes.MAT_SAND))
    e.set_planes([[0.0, 1.0, 0.0, -float(B.FLOOR)]], 0.4)
    return e


def frame_aos(e, pool, idx, alive, L, substeps):
    e.upload_aos(pool, idx[:alive], L)
    e.substep(substeps)
    return e.download_aos(pool, idx[:alive], L)


def frame_fieldwise(e, pool, idx, alive, L, substeps):
    f = pool.view(np.float32).reshape(-1, L.stride // 4)
    cols = columns(L)
    slots = idx[:alive].astype(np.int64)
    rows = f[slots]                                         # gather
    st = {k: rows[:, c] for k, c in cols.items()}
    e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"])
    e.substep(substeps)
    got = e.download(sort_by_id=False)
    s = slots[got["id"].astype(np.int64)]                   # scatter back by id (id = position in the upload)
    for k, c in cols.items():
        f[s[:, None], np.atleast_1d(c)] = got[k].reshape(len(s), -1)
    keep = np.zeros(alive, bool)
    keep[got["id"]] = True
    n = int(keep.sum())
    idx[:n] = idx[:alive][keep]                             # survivors in id order, as clear_boundary_particles leaves them
    return n


def run_leg(kind, res, st, dt, pool, idx, L, frames, substeps):
    n = len(st["x"])
    pool[:] = 0
    fill(pool, st, L)
    idx[:] = np.arange(n, dtype=np.uint32)
    e = engine(res, dt)
    try:
        alive, times = n, []
        if kind == "substeps":
            e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"])
        for fr in range(frames + 1):
            t0 = time.perf_counter()
            if kind == "substeps":
                e.substep(substeps)
                e.synchronize()
                alive = e.num_particles()
            else:
                alive = (frame_aos if kind == "aos" else frame_fieldwise)(e, pool, idx, alive, L, substeps)
            if fr > 0:   # frame 0 warms the staging buffers and captures the graphs
                times.append(time.perf_counter() - t0)
        sec = float(np.median(times))
        out = dict(leg=kind, alive=int(alive), updates_per_s_M=alive * substeps / sec / 1e6, frame_seconds=sec,
                   frame_seconds_all=[float(t) for t in times])
        slots = len(pool) // L.stride
        if kind == "aos":
            w = window(L)
            out.update(window=list(w), bytes_h2d=(w[1] - w[0]) * slots + 4 * n, bytes_d2h=(w[1] - w[0]) * slots + 4 * alive)
        elif kind == "fieldwise":
            out.update(bytes_h2d=FIELDWISE_UP * n, bytes_d2h=FIELDWISE_DOWN * n)
        return out
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--substeps", type=int, default=500)
    ap.add_argument("--sizes", default="1024,2048")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropin_2d.py measures on a CUDA device; none is visible")
    L = layout()
    line = {"metric": "mpm2d_dropin_mupdates_per_s", "unit": "M particle-updates/s", "substeps_per_frame": args.substeps, "frames": args.frames,
            "card": B.card(0), "sizes": []}
    for res in (int(s) for s in args.sizes.split(",")):
        st, dt = B.column(res)
        n = len(st["x"])
        pool_t = torch.zeros(n * L.stride, dtype=torch.uint8, pin_memory=True)
        idx_t = torch.empty(n, dtype=torch.int32, pin_memory=True)
        pool, idx = pool_t.numpy(), idx_t.numpy().view(np.uint32)
        legs, ends = [], {}
        for kind in ("aos", "fieldwise", "substeps"):
            legs.append(run_leg(kind, res, st, dt, pool, idx, L, args.frames, args.substeps))
            if kind != "substeps":
                ends[kind] = (pool.copy(), idx[: legs[-1]["alive"]].copy())
        same = np.array_equal(ends["aos"][0], ends["fieldwise"][0]) and np.array_equal(ends["aos"][1], ends["fieldwise"][1])
        assert same, "the AoS and field-wise legs left different pools"
        line["sizes"].append(dict(res=[res, res], particles=n, dt=dt, pools_identical=same, legs=legs))
        del pool_t, idx_t
    line["value"] = line["sizes"][0]["legs"][0]["updates_per_s_M"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
