"""Edits of the resident set on z-slab ranks, on the flagship workload (sand256: 8 M sand particles, 256^3) split over W = 2
and 4 slabs in ONE process on ONE GPU, exchanging through the engine's peer-memory path.  This times the edit path of a
rank (mpmb_append_owned_particles, mpmb_delete_owned_inside_levelset through slab.py), not multi-GPU scaling.

    python bench_slab_edit.py [--warmup 20]

Per W, three copies of the scene make the same edits after the same substeps: the slab ranks with the device edits, the
slab ranks with the only edit possible before them (download every rank, edit on the host, upload every rank again, which
renumbers the ids), and one engine with mpmb_append_particles / mpmb_delete_inside_levelset.  Edits: append 1 % and 10 %
of the set (lattice layers above the column), then delete below a plane through the column.  Prints one JSON line: the
card and its power limit (read in the same run), the wall time of each edit with a device synchronise, the first substep
after it and a steady one (CUDA events around the interleaved stages of all ranks), and whether the device edits leave the
same live set as the single engine (ids and positions) and as the round trip (positions: it renumbers).  Needs a CUDA
device: without one it exits with an error and measures nothing."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_resident_edit import card, same_live_set  # noqa: E402

KEYS = ("x", "v", "mass", "vol", "F", "b", "ps", "group")


class Slabs:
    """W z-slab engines of the seeded scene, peer-connected inside this process; one substep = the interleaved stages."""

    def __init__(self, cfg, world):
        from taichi_mpm_b200 import capi, slab
        sc, m = cfg["scene"], cfg["meta"]
        dx = sc["dx"]
        # tile layer of every lattice particle's base node, without the 8 M positions: per cell layer half the corners
        # (offset 0.25) have their base node in the layer below, half (0.75) in the layer itself
        kz = np.arange(m["lo"][2], m["hi"][2])
        per = (m["hi"][0] - m["lo"][0]) * (m["hi"][1] - m["lo"][1]) * 4
        tz = np.repeat(np.concatenate([(kz - 1) >> 2, kz >> 2]), per)
        self.cuts = slab.slab_partition(tz, slab.tile_layers(m["res"]), world)
        self.eng = []
        for rank, (z0, z1) in enumerate(self.cuts):
            e = capi.Engine(sc["res"], dx, sc["dt"], sc["gravity"], sc["particle_gravity"], True, rank=rank, world=world, tile_z0=z0, tile_z1=z1)
            e.set_material(0, m["kind"], sc["mat_params"][0])
            e.set_planes(sc["planes"], sc["friction"])
            e.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
            self.eng.append(e)
        for r in range(world - 1):
            for k in (0, 1):
                self.eng[r].xchg_connect(k, 1, ptr=self.eng[r + 1].xchg_buffer(k, 0))
                self.eng[r + 1].xchg_connect(k, 0, ptr=self.eng[r].xchg_buffer(k, 1))
        self.faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < world] for r in range(world)]

    def substep(self, n=1):
        for _ in range(n):
            for e in self.eng:
                e.sort_particles_and_populate_grid(); e.rasterize()
            for op in ("halo_send", "halo_recv"):
                for r, e in enumerate(self.eng):
                    for f in self.faces[r]:
                        getattr(e, op)(f)
            for e in self.eng:
                e.resample()
            for op in ("migrate_send", "migrate_recv"):
                for r, e in enumerate(self.eng):
                    for f in self.faces[r]:
                        getattr(e, op)(f)

    def download(self):
        parts = [e.download() for e in self.eng]
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def round_trip(self, edit):
        """Every rank to the host, edited there (edit(rank, fields)), every rank uploaded again with fresh ids."""
        base = 0
        for r, e in enumerate(self.eng):
            d = e.download()
            h = edit(r, {k: d[k] for k in KEYS})
            e.set_id_base(base)
            e.upload(*(h[k] for k in KEYS))
            base += len(h["x"])

    def close(self):
        for e in self.eng:
            e.close()


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def substep_ms(step):
    """(first substep after the edit, the next one), CUDA events on the stream every engine uses."""
    import torch
    out = []
    for _ in range(2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def by_id(d):
    o = np.argsort(d["id"], kind="stable")
    return {k: v[o] for k, v in d.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20, help="substeps before the first edit")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_slab_edit.py needs a CUDA device (an H100); nothing was measured")
    from taichi_mpm_b200 import capi, mpm as mpm_mod, scenes, slab
    name, limit = card()
    cfg = scenes.config("sand256", 1.0, state=False)
    sc, m = cfg["scene"], cfg["meta"]
    res, dx = m["res"], sc["dx"]
    out = {"metric": "slab_resident_set_edit", "workload": "sand256", "gpu": name, "power_limit_w": limit, "warmup_substeps": args.warmup,
           "note": "W slabs in one process on one GPU (peer-memory path): times the edit path, not multi-GPU scaling"}
    ycut = 0.5 * (m["lo"][1] + m["hi"][1])
    cut = np.array([[0.0, 1.0, 0.0, -ycut]], np.float32)
    ls = mpm_mod.LevelSet((res,) * 3, dx)
    ls.add_plane((0.0, 1.0, 0.0), -ycut * dx)
    for world in (2, 4):
        dev, old = Slabs(cfg, world), Slabs(cfg, world)
        one = capi.Engine(sc["res"], dx, sc["dt"], sc["gravity"], sc["particle_gravity"], True)
        one.set_material(0, m["kind"], sc["mat_params"][0])
        one.set_planes(sc["planes"], sc["friction"])
        one.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
        for s in (dev, old):
            s.substep(args.warmup)
        one.substep(args.warmup)
        torch.cuda.synchronize()
        res_w = {"cuts": dev.cuts}
        y0 = 120
        for label, layers in (("append_1pct", 1), ("append_10pct", 10)):
            # lattice layers above the column: 100 x layers x 100 cells, 80 000 particles per layer
            x, mass, vol = scenes.lattice_block(res, (m["lo"][0], y0, m["lo"][2]), (m["hi"][0], y0 + layers, m["hi"][2]), m["density"], dx=dx)
            y0 += layers + 2
            st = scenes.make_state(x, mass, vol, m["kind"])
            new = {k: st[k] for k in KEYS}
            n0 = sum(e.num_particles() for e in dev.eng)
            first = max(slab.global_id_end(e) for e in dev.eng)
            kept, t_dev = timed(lambda: [slab.append_particles(e, new, first) for e in dev.eng])
            tz = slab.base_tile_z(new["x"][:, 2], dx)
            _, t_old = timed(lambda: old.round_trip(lambda r, h: {k: np.concatenate([h[k], new[k][(tz >= dev.cuts[r][0]) & (tz < dev.cuts[r][1])]]) for k in h}))
            assert one.append(*(new[k] for k in KEYS)) == first
            res_w[label] = {"n_resident": n0, "n_new": len(new["x"]), "first_id": first, "kept_per_rank": kept, "device_ms": t_dev, "round_trip_ms": t_old}
        torch.cuda.synchronize()
        a, b, c = dev.download(), old.download(), by_id(one.download())
        same, dpos = same_live_set(a, b)
        res_w["after_appends"] = {"same_live_set_as_round_trip": same, "round_trip_max_x_diff": dpos}
        a = by_id(a)
        res_w["after_appends"].update(ids_equal_single_engine=bool(np.array_equal(a["id"], c["id"])),
                                      max_x_diff_single_engine=float(np.abs(a["x"] - c["x"]).max()) if len(a["id"]) == len(c["id"]) else None)
        s_dev, s_old = substep_ms(dev.substep), substep_ms(old.substep)
        one.substep(2)
        res_w["after_appends"].update(first_substep_ms=s_dev[0], steady_substep_ms=s_dev[1], round_trip_first_substep_ms=s_old[0])
        for s in (dev, old):
            for e in s.eng:
                e.set_planes(cut, sc["friction"])
        one.set_planes(cut, sc["friction"])
        torch.cuda.synchronize()
        n0 = sum(e.num_particles() for e in dev.eng)
        n_del, t_dev = timed(lambda: [slab.delete_inside_levelset(e) for e in dev.eng])

        def keep_outside(r, h):
            keep = ~(ls.sample(h["x"].astype(np.float64) / dx) < 0)
            return {k: np.ascontiguousarray(v[keep]) for k, v in h.items()}

        _, t_old = timed(lambda: old.round_trip(keep_outside))
        n_one = one.delete_inside_levelset()
        a, b, c = dev.download(), old.download(), by_id(one.download())
        same_rt, dpos_rt = same_live_set(a, b)   # the round trip's rows were uploaded in another order two substeps earlier
        a = by_id(a)
        s_dev, s_old = substep_ms(dev.substep), substep_ms(old.substep)
        res_w["delete_plane"] = {"n_resident": n0, "n_deleted_per_rank": n_del, "n_deleted_single_engine": n_one, "device_ms": t_dev,
                                 "round_trip_ms": t_old, "first_substep_ms": s_dev[0], "steady_substep_ms": s_dev[1],
                                 "round_trip_first_substep_ms": s_old[0], "same_live_set_as_round_trip": same_rt, "round_trip_max_x_diff": dpos_rt, "n_live": len(a["x"]), "round_trip_n_live": len(b["x"]),
                                 "ids_equal_single_engine": bool(np.array_equal(a["id"], c["id"])),
                                 "max_x_diff_single_engine": float(np.abs(a["x"] - c["x"]).max()) if len(a["id"]) == len(c["id"]) else None}
        out["W%d" % world] = res_w
        dev.close(); old.close(); one.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
