"""Rigid-coupled substeps on z slabs: bench_rigid.py's scene (128^3 grid, 1.0 M jelly particles, a scripted paddle, a free box,
a floor plane with the rigid-body level-set collision), cut into W = 1, 2 and 4 slabs through the block and the paddle, all
ranks in one process on one GPU, exchanging through peer memory (halo, migration, impulse mailboxes) on one stream.

    python bench_slab_rigid.py [--steps 100] [--warmup 10] [--res 128]
    python bench_slab_rigid.py --procs [--steps 100]     # >= 2 GPUs: one process per GPU, mpmb_substep with IPC peers

Prints one JSON line: the card and its power limit (read in the same run); per W the per-rank maximum of each stage's time per
substep summed over the stages (a proxy for a W-GPU substep: the ranks run one after another here, so wall time is not the
measure), the time of the two impulse reductions per substep, and the body and particle differences against W = 1.  With
--procs: the wall time per substep of W = #GPUs processes.  Needs a CUDA device."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_rigid  # noqa: E402


def parts(res, nsub):
    """Particles (ids 0..n-1), bodies, motion rows and an nsub-entry script table of bench_rigid's scene."""
    from taichi_mpm_b200 import capi
    m = bench_rigid.scene(res)
    st = m.engine.download()
    rec = m._rigid_records()
    rows = [{}] + [b.motion_record() for b in m.rigids]
    h, t = np.float32(m.base_delta_t), np.float32(m.current_t)
    clocks = []
    for _ in range(nsub):
        clocks.append(float(t) + float(h))
        t = np.float32(t + h)
    table = np.zeros((nsub, len(m.rigids) + 1, capi.RIGID_SCRIPT_STRIDE))
    for k, b in enumerate(m.rigids):
        if b.pos_func is not None or b.rot_func is not None:
            table[:, k + 1] = b.script_poses(clocks, float(h))
    m.engine.close()
    return m, st, rec, rows, table


def cuts_for(st, m, world):
    from taichi_mpm_b200 import slab
    tz = slab.base_tile_z(st["x"][:, 2], m.delta_x)
    return slab.slab_partition(tz, slab.tile_layers(m.res[2]), world)


def engines(m, st, rec, rows, table, world, device=0, stream=None):
    from taichi_mpm_b200 import capi
    n = len(st["x"])
    out = []
    for r, (z0, z1) in enumerate(cuts_for(st, m, world)):
        e = capi.Engine(m.res, m.delta_x, m.base_delta_t, m.gravity, True, True, device=device, capacity=2 * n if world > 1 else 0, rank=r,
                        world=world, tile_z0=z0, tile_z1=z1, migrate_capacity=1 << 16)
        if stream is not None:
            e.set_stream(stream)
        for g, (kind, prm) in enumerate(m._groups):
            e.set_material(g, kind, prm)
        e.set_planes(m._levelset.planes_grid_units(), m._levelset.friction)
        e.append_owned(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"], first_id=0)
        e.set_rigid(rec)
        e.set_rigid_motion(rows, levelset_collision=True)
        e.set_rigid_script(table)
        out.append(e)
    for r in range(world - 1):
        for k in (0, 1):
            out[r].xchg_connect(k, 1, ptr=out[r + 1].xchg_buffer(k, 0))
            out[r + 1].xchg_connect(k, 0, ptr=out[r].xchg_buffer(k, 1))
    for r in range(world):
        for j in range(world):
            if j != r:
                out[r].rigid_connect(j, ptr=out[j].rigid_mailbox())
    return out


class Timer:
    """CUDA events on the shared stream around one piece of work; elapsed times are read once at the end."""

    def __init__(self, torch):
        self.torch, self.ev = torch, []

    def __call__(self, key, fn):
        a, b = self.torch.cuda.Event(enable_timing=True), self.torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        self.ev.append((key, a, b))

    def totals(self):
        self.torch.cuda.synchronize()
        out = {}
        for key, a, b in self.ev:
            out[key] = out.get(key, 0.0) + a.elapsed_time(b)
        return out


def substep(eng, tm=None):
    """One staged substep of every rank; with a Timer, stage k of rank r is timed as ('stage', k, r), the reductions as 'reduce'."""
    W = len(eng)
    run = tm if tm is not None else (lambda key, fn: fn())
    faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < W] for r in range(W)]

    def reduce():
        for e in eng:
            e.rigid_send()
        for e in eng:
            e.rigid_recv()
    if W == 1:
        run(("stage", 0, 0), lambda: (eng[0].sort_particles_and_populate_grid(), eng[0].rasterize()))
        run(("stage", 1, 0), eng[0].resample)
        return
    for r, e in enumerate(eng):
        run(("stage", 0, r), lambda e=e: (e.sort_particles_and_populate_grid(), e.rasterize()))
    run("reduce", reduce)
    for r, e in enumerate(eng):
        run(("stage", 1, r), lambda r=r, e=e: [e.halo_send(f) for f in faces[r]])
    for r, e in enumerate(eng):
        run(("stage", 2, r), lambda r=r, e=e: ([e.halo_recv(f) for f in faces[r]], e.resample()))
    run("reduce", reduce)
    for r, e in enumerate(eng):
        run(("stage", 3, r), lambda r=r, e=e: [e.migrate_send(f) for f in faces[r]])
    for r, e in enumerate(eng):
        run(("stage", 4, r), lambda r=r, e=e: [e.migrate_recv(f) for f in faces[r]])


def end_state(eng, nb):
    parts_ = [e.download() for e in eng]
    u = {k: np.concatenate([p[k] for p in parts_]) for k in ("id", "x", "v")}
    o = np.argsort(u["id"])
    return {k: v[o] for k, v in u.items()}, eng[0].get_rigid_state(nb)


def one_process(a):
    import torch
    m, st, rec, rows, table = parts(a.res, a.warmup + a.steps)
    nb = len(rec["inv_mass"])
    stream = torch.cuda.current_stream().cuda_stream
    res, ref = {}, None
    for world in (1, 2, 4):
        eng = engines(m, st, rec, rows, table, world, stream=stream)
        for _ in range(a.warmup):
            substep(eng)
        tm = Timer(torch)
        for _ in range(a.steps):
            substep(eng, tm)
        tot = tm.totals()
        stages = sorted({k[1] for k in tot if k != "reduce"})
        proxy = sum(max(tot[("stage", s, r)] for r in range(world) if ("stage", s, r) in tot) for s in stages) / a.steps
        red = tot.get("reduce", 0.0) / a.steps
        u, body = end_state(eng, nb)
        for e in eng:
            e.close()
        if ref is None:
            ref = (u, body)
        assert np.array_equal(u["id"], ref[0]["id"])
        res["W%d" % world] = dict(cuts=cuts_for(st, m, world), rank_max_stage_ms_per_substep=proxy + red, reductions_ms_per_substep=red,
                                  body_position_diff=float(np.abs(body["position"] - ref[1]["position"]).max()),
                                  body_velocity_diff=float(np.abs(body["velocity"] - ref[1]["velocity"]).max()),
                                  particle_x_diff=float(np.abs(u["x"] - ref[0]["x"]).max()),
                                  particle_v_diff_rel=float(np.abs(u["v"] - ref[0]["v"]).max() / max(np.abs(ref[0]["v"]).max(), 1e-30)))
    return res


def _proc(rank, world, port, a, q):
    import torch
    import torch.distributed as dist
    from taichi_mpm_b200 import capi, slab
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    m, st, rec, rows, table = parts(a.res, a.warmup + a.steps)
    z0, z1 = cuts_for(st, m, world)[rank]
    e = capi.Engine(m.res, m.delta_x, m.base_delta_t, m.gravity, True, True, device=rank, capacity=2 * len(st["x"]), rank=rank, world=world,
                    tile_z0=z0, tile_z1=z1, migrate_capacity=1 << 16)
    for g, (kind, prm) in enumerate(m._groups):
        e.set_material(g, kind, prm)
    e.set_planes(m._levelset.planes_grid_units(), m._levelset.friction)
    e.append_owned(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"], first_id=0)
    e.set_rigid(rec)
    e.set_rigid_motion(rows, levelset_collision=True)
    e.set_rigid_script(table)
    slab.connect_peers(e, rank, world, dist)
    e.substep(a.warmup)
    e.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    e.substep(a.steps)
    e.synchronize()
    dist.barrier()
    q.put((rank, (time.perf_counter() - t0) * 1e3 / a.steps))
    e.close()
    dist.destroy_process_group()


def multi_process(a):
    import socket
    import torch
    import torch.multiprocessing as mp
    world = torch.cuda.device_count()
    if world < 2:
        raise SystemExit("--procs needs at least 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_proc, args=(r, world, port, a, q)) for r in range(world)]
    for p in procs:
        p.start()
    ms = dict(q.get(timeout=1800) for _ in range(world))
    for p in procs:
        p.join()
    return {"W%d_procs" % world: dict(wall_ms_per_substep=max(ms.values()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--procs", action="store_true")
    a = ap.parse_args()
    name, limit = bench_rigid.card()
    res = multi_process(a) if a.procs else one_process(a)
    print(json.dumps(dict(bench="slab_rigid", card=name, power_limit_w=limit, res=a.res, steps=a.steps, warmup=a.warmup, **res)))


if __name__ == "__main__":
    main()
