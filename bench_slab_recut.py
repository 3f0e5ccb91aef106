"""Re-cut of the z slabs on the flagship workload (sand256: 8 M sand particles, 256^3) split over W = 2 and 4 slabs in ONE
process on ONE GPU, exchanging through the engine's peer-memory path, as bench_slab_edit.py does.

    python bench_slab_recut.py [--develop 20000] [--steps 20]        one process, one GPU
    python bench_slab_recut.py --procs [--develop 20000] [--steps 20] one process per visible GPU (>= 2), NCCL

The cuts are taken from the resting column (slab.slab_partition of the seeded lattice, as bench.py --gpus N takes them).
Two ways to unbalance them, each measured before and after slab-style re-cut (mpmb_layer_counts / mpmb_recut_pack /
mpmb_recut_apply):
  (a) the developed collapse: one engine runs `--develop` substeps from the resting column (bench.py's default), its state
      is split over the slabs by the resting cuts;
  (b) a 10 % append into the region of slab 0 (a lattice block beside the column, every base node below the first cut).
Per case: per-rank live counts; per-rank stage time per substep from CUDA events around that rank's own stages
(mpmb_set_profiling) and its maximum over the ranks; the re-cut's wall time with a device synchronise against the only
re-cut possible before it (download every rank, new engines with the new cuts, upload, connect the peers); and whether the
union of the ranks by id is bit-identical across the re-cut.  In one process on one GPU the ranks' stages run one after
another, so the maximum over ranks is a PROXY for the critical path of a W-GPU substep, not a multi-GPU time.

--procs runs W = the number of visible GPUs, one process each, and reports the wall time of mpmb_substep (peer-memory
path) per substep before and after slab.rebalance.  Each mode prints one JSON line with the card and its power limit, read
in the same run.  Needs a CUDA device: without one it exits with an error and measures nothing."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_resident_edit import card  # noqa: E402

KEYS = ("x", "v", "mass", "vol", "F", "b", "ps", "group")


def resting_cuts(m, world):
    """Cuts of the resting column: per cell layer half the corners (offset 0.25) have their base node in the layer below,
    half (0.75) in the layer itself (bench_slab_edit.py)."""
    from taichi_mpm_b200 import slab
    kz = np.arange(m["lo"][2], m["hi"][2])
    per = (m["hi"][0] - m["lo"][0]) * (m["hi"][1] - m["lo"][1]) * 4
    tz = np.repeat(np.concatenate([(kz - 1) >> 2, kz >> 2]), per)
    return slab.slab_partition(tz, slab.tile_layers(m["res"]), world)


def make_engine(cfg, rank=0, world=1, z=(0, 0), device=0):
    from taichi_mpm_b200 import capi
    sc, m = cfg["scene"], cfg["meta"]
    e = capi.Engine(sc["res"], sc["dx"], sc["dt"], sc["gravity"], sc["particle_gravity"], True, device=device, rank=rank, world=world,
                    tile_z0=z[0], tile_z1=z[1])
    e.set_material(0, m["kind"], sc["mat_params"][0])
    e.set_planes(sc["planes"], sc["friction"])
    return e


class Slabs:
    """W z-slab engines, peer-connected inside this process; one substep = the interleaved stages of all ranks."""

    def __init__(self, cfg, cuts, state=None):
        self.cfg, self.cuts, self.world = cfg, list(cuts), len(cuts)
        m = cfg["meta"]
        self.eng = [make_engine(cfg, r, self.world, z) for r, z in enumerate(cuts)]
        if state is None:
            for e in self.eng:
                e.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
        else:
            self.upload(state)
        self.connect()

    def upload(self, d):
        from taichi_mpm_b200 import slab
        tz = slab.base_tile_z(d["x"][:, 2], self.cfg["scene"]["dx"])
        base = 0
        for e, (z0, z1) in zip(self.eng, self.cuts):
            sel = np.nonzero((tz >= z0) & (tz < z1))[0]
            e.set_id_base(base)
            e.upload(*(d[k][sel] for k in KEYS))
            base += len(sel)

    def connect(self):
        for r in range(self.world - 1):
            for k in (0, 1):
                self.eng[r].xchg_connect(k, 1, ptr=self.eng[r + 1].xchg_buffer(k, 0))
                self.eng[r + 1].xchg_connect(k, 0, ptr=self.eng[r].xchg_buffer(k, 1))
        self.faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < self.world] for r in range(self.world)]

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

    def stage_ms(self, steps):
        """Per rank: device milliseconds per substep summed over its own stages (CUDA events on its stream)."""
        for e in self.eng:
            e.get_profile(reset=True)
            e.set_profiling(True)
        self.substep(steps)
        out = []
        for e in self.eng:
            ms, _ = e.get_profile(reset=True)
            e.set_profiling(False)
            out.append(sum(ms) / steps)
        return out

    def union(self):
        parts = [e.download() for e in self.eng]
        d = {k: np.concatenate([p[k] for p in parts]) for k in ("id",) + KEYS}
        o = np.argsort(d["id"], kind="stable")
        return {k: v[o] for k, v in d.items()}

    def recut(self):
        """slab.rebalance's choreography for the engines of one process (device buffers, one pack and one apply per rank)."""
        import torch
        from taichi_mpm_b200 import capi, slab
        hist = sum(e.layer_counts() for e in self.eng)
        new = slab.partition_counts(hist, self.world)
        if new == self.cuts:   # as slab.rebalance: balanced already, nothing moves
            return 0
        flat = [0] + [z1 for _, z1 in new]
        packs = []
        for e in self.eng:
            counts = e.recut_pack(flat)
            b = torch.empty(int(counts.sum()) * capi.RECORD_BYTES, dtype=torch.uint8, device="cuda")
            e.recut_pack(flat, b)
            packs.append((counts, b))
        rb = capi.RECORD_BYTES
        for r, e in enumerate(self.eng):
            pieces = [b[int(c[:r].sum()) * rb:int(c[:r + 1].sum()) * rb] for c, b in packs if c[r]]
            e.recut_apply(new[r][0], new[r][1], torch.cat(pieces) if pieces else None, sum(int(c[r]) for c, _ in packs))
        self.cuts = new
        return sum(int(c.sum()) for c, _ in packs)

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


def measure(S, cfg, steps):
    """Before / after the re-cut: counts, per-rank stage time, the re-cut against the round trip, the bitwise check."""
    import torch
    res = {"cuts_before": [list(c) for c in S.cuts], "live_before": [e.num_particles() for e in S.eng]}
    S.substep(2)
    res["stage_ms_before"] = S.stage_ms(steps)
    before = S.union()
    moved, t_recut = timed(S.recut)
    after = S.union()
    res["bitwise_identical_by_id"] = bool(len(before["id"]) == len(after["id"]) and
                                          all(np.array_equal(before[k].view(np.uint8), after[k].view(np.uint8)) for k in before))
    res.update(cuts_after=[list(c) for c in S.cuts], live_after=[e.num_particles() for e in S.eng], rows_moved=moved, recut_ms=t_recut)
    S.substep(2)
    res["stage_ms_after"] = S.stage_ms(steps)
    for k in ("before", "after"):
        res["max_rank_stage_ms_" + k] = max(res["stage_ms_" + k])
    # the re-cut possible before: every rank to the host, new engines with the new cuts, upload, peers connected
    cuts = list(S.cuts)
    del before, after

    def round_trip():
        d = S.union()
        T = Slabs(cfg, cuts, state=d)
        return T

    T, t_rt = timed(round_trip)
    T.close()
    res["round_trip_ms"] = t_rt
    torch.cuda.synchronize()
    return res


def one_process(args):
    import torch
    from taichi_mpm_b200 import scenes
    name, limit = card()
    cfg = scenes.config("sand256", 1.0, state=False)
    m = cfg["meta"]
    out = {"metric": "slab_recut", "workload": "sand256", "gpu": name, "power_limit_w": limit, "develop_substeps": args.develop,
           "timed_substeps": args.steps,
           "note": "W slabs in one process on one GPU (peer-memory path); max_rank_stage_ms is a proxy for the critical path of "
                   "a W-GPU substep, not a multi-GPU time"}
    # (a) the developed collapse, from one engine with graph replay
    one = make_engine(cfg)
    one.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
    one.substep(args.develop)
    developed = one.download()
    one.close()
    for world in (2, 4):
        S = Slabs(cfg, resting_cuts(m, world), state=developed)
        out["developed_W%d" % world] = measure(S, cfg, args.steps)
        S.close()
    del developed
    # (b) a 10 % append into the region of slab 0, on the resting column
    from taichi_mpm_b200 import slab
    for world in (2, 4):
        S = Slabs(cfg, resting_cuts(m, world))
        S.substep(2)
        n0 = sum(e.num_particles() for e in S.eng)
        z_hi = 4 * S.cuts[0][1] - 1
        nx, nz = m["hi"][0] - m["lo"][0], z_hi - m["lo"][2]
        layers = int(np.ceil(0.1 * n0 / (8 * nx * nz)))
        y0 = m["hi"][1] + 2
        x, mass, vol = scenes.lattice_block(m["res"], (m["lo"][0], y0, m["lo"][2]), (m["hi"][0], y0 + layers, z_hi), m["density"], dx=cfg["scene"]["dx"])
        st = scenes.make_state(x, mass, vol, m["kind"])
        first = max(slab.global_id_end(e) for e in S.eng)
        kept = [slab.append_particles(e, {k: st[k] for k in KEYS}, first) for e in S.eng]
        r = measure(S, cfg, args.steps)
        r.update(appended=len(x), appended_kept_per_rank=kept)
        out["append10_W%d" % world] = r
        S.close()
    torch.cuda.synchronize()
    print(json.dumps(out))


def _proc(rank, world, port, args, q):
    import torch
    import torch.distributed as dist
    from taichi_mpm_b200 import scenes, slab
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    cfg = scenes.config("sand256", 1.0, state=False)
    m = cfg["meta"]
    e = make_engine(cfg, rank, world, resting_cuts(m, world)[rank], device=rank)
    e.set_stream(torch.cuda.current_stream().cuda_stream)
    e.seed_lattice(m["lo"], m["hi"], m["vol"], m["mass"], jitter=m["jitter"], seed=m["seed"])
    slab.connect_peers(e, rank, world, dist)
    e.substep(args.develop)

    def wall():
        e.substep(2)
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        e.substep(args.steps)
        torch.cuda.synchronize()
        dist.barrier()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    res = {"live_before": e.num_particles(), "substep_ms_before": wall()}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    old, new, moved = slab.rebalance(e, rank, world, dist)
    torch.cuda.synchronize()
    res.update(recut_ms=(time.perf_counter() - t0) * 1e3, cuts_before=old, cuts_after=new, rows_moved=moved, live_after=e.num_particles(),
               substep_ms_after=wall())
    q.put((rank, res))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


def procs(args):
    import socket
    import torch
    import torch.multiprocessing as mp
    world = torch.cuda.device_count()
    if world < 2:
        sys.exit("--procs needs at least 2 visible GPUs; nothing was measured")
    name, limit = card()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_proc, args=(r, world, port, args, q)) for r in range(world)]
    for p in ps:
        p.start()
    ranks = dict(q.get() for _ in range(world))
    for p in ps:
        p.join()
    print(json.dumps({"metric": "slab_recut_procs", "workload": "sand256", "gpu": name, "power_limit_w": limit, "world": world,
                      "develop_substeps": args.develop, "timed_substeps": args.steps, "ranks": [ranks[r] for r in range(world)]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--develop", type=int, default=20000, help="substeps of the collapse before case (a) (bench.py's sand256 default)")
    ap.add_argument("--steps", type=int, default=20, help="timed substeps before and after each re-cut")
    ap.add_argument("--procs", action="store_true", help="one process per visible GPU, NCCL re-cut, mpmb_substep wall time")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_slab_recut.py needs a CUDA device (an H100); nothing was measured")
    (procs if args.procs else one_process)(args)


if __name__ == "__main__":
    main()
