"""z-slab multi-GPU driver: one process per GPU, torch.distributed for the plumbing.

A rank owns the particles whose base node lies in tile layers [z0, z1) (tiles are 4 nodes thick,
cuts only at tile boundaries).  Per substep the engine (C-ABI, include/mpmb.h) does all device work;
this module only moves two kinds of device buffers between ring neighbours:

  after rasterize : boundary-layer arenas (partial sums of grid momentum/mass) both ways,
                    unpacked by the neighbour as ghost tiles before resample;
  after resample  : particles that left the slab through a face, appended by the neighbour.

With rigid coupling every rank also takes part in two all-gathers per substep: after each transfer the ranks' partial sums
of the bodies' impulses (engine.rigid_impulse_bytes() each), which every engine sums in rank order and applies.

Messages have a fixed size agreed at start-up (engine.halo_bytes()/migrate_bytes()), so the host
never waits for a device-side count.  No collective is on the data path: point-to-point only.
"""
import numpy as np


def tile_layers(res_z):
    """Number of tile layers of the engine's tile grid along an axis of `res_z` cells."""
    return (res_z + 1 + 3) // 4 + 1


def base_tile_z(z, dx):
    """Tile layer of the base node, with the engine's float32 arithmetic (src/kernel.h:119-121)."""
    X = (np.asarray(z, np.float32) * np.float32(1.0 / np.float32(dx))).astype(np.float32)
    return (X - np.float32(0.5)).astype(np.int32) >> 2


def layer_histogram(tile_z, n_layers):
    """Particles per tile layer of [0, n_layers), from the tile layer of every particle."""
    return np.bincount(np.asarray(tile_z, np.int64), minlength=n_layers)[:n_layers]


def partition_counts(hist, world):
    """Cuts the tile layers of a particle histogram (hist[l] = particles in layer l) into `world` contiguous slabs with
    balanced particle counts.  Returns [(z0, z1)] * world; every slab has >= 1 layer and the cuts are placed by the prefix
    sum of the histogram over the occupied extent (column-collapse scenes occupy a small part of the domain, SURVEY §8e)."""
    hist = np.asarray(hist, np.float64)
    n_layers = len(hist)
    cum = np.cumsum(hist)
    total = cum[-1] if len(cum) else 0.0
    cuts = [0]
    for r in range(1, world):
        if total > 0:
            z = int(np.searchsorted(cum, total * r / world, side="left")) + 1
        else:
            z = n_layers * r // world
        z = max(z, cuts[-1] + 1)
        z = min(z, n_layers - (world - r))
        cuts.append(z)
    cuts.append(n_layers)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def slab_partition(tile_z, n_layers, world):
    """partition_counts of the histogram of tile_z (the tile layer of every particle)."""
    return partition_counts(layer_histogram(tile_z, n_layers), world)


def _refuse_2d(engine):
    """z-slabs split the z axis of an MPM<3> engine; a 2-D engine (capi.Engine2D) has none."""
    if getattr(getattr(engine, "cfg", None), "dim", 0) == 2:
        raise ValueError("z-slab runs are MPM<3> only: a 2-D engine runs on one GPU")


class EngineAdapter:
    """Binds torch buffers to the pointer-based exchange calls of capi.Engine."""

    def __init__(self, engine):
        _refuse_2d(engine)
        self.e = engine

    def halo_bytes(self):
        return self.e.halo_bytes()

    def migrate_bytes(self):
        return self.e.migrate_bytes()

    def sort(self):
        self.e.sort_particles_and_populate_grid()

    def rasterize(self):
        self.e.rasterize()

    def resample(self):
        self.e.resample()

    def rasterize_part(self, part):
        self.e.rasterize_part(part)

    def resample_part(self, part):
        self.e.resample_part(part)

    def halo_pack(self, face, buf):
        self.e.halo_pack(face, buf.data_ptr())

    def halo_unpack(self, face, buf):
        self.e.halo_unpack(face, buf.data_ptr())

    def migrate_pack(self, face, buf):
        self.e.migrate_pack(face, buf.data_ptr())

    def migrate_unpack(self, face, buf):
        self.e.migrate_unpack(face, buf.data_ptr())

    def share_id_end(self, dist):
        share_id_end(self.e, dist)

    def rigid_on(self):
        return self.e.rigid_impulse_bytes() > 0 and getattr(self.e, "rigid_coupled", False)

    def rigid_impulse_bytes(self):
        return self.e.rigid_impulse_bytes()

    def rigid_impulse_pack(self, buf):
        self.e.rigid_impulse_pack(buf.data_ptr())

    def rigid_impulse_apply(self, buf):
        self.e.rigid_impulse_apply(buf.data_ptr())


class SlabRunner:
    """Runs substeps of one slab and exchanges with the ring neighbours (rank-1 below, rank+1 above)."""

    def __init__(self, adapter, rank, world, device, dist=None, group=None, overlap=False):
        import torch
        self.torch = torch
        self.a = adapter
        self.rank, self.world = rank, world
        self.dist = dist
        self.group = group
        # overlap=True splits every tile kernel into boundary-layer and interior launches and flies the
        # halo during the interior work.  The partial launches can cost more than the NVLink time they
        # hide, so the plain schedule is the default.
        self.overlap = overlap
        self.has_lo = rank > 0
        self.has_hi = rank < world - 1
        hb, mb = adapter.halo_bytes(), adapter.migrate_bytes()
        mk = lambda n: torch.empty(max(int(n), 16), dtype=torch.uint8, device=device)
        self.halo_send = [mk(hb), mk(hb)]
        self.halo_recv = [mk(hb), mk(hb)]
        self.mig_send = [mk(mb), mk(mb)]
        self.mig_recv = [mk(mb), mk(mb)]
        self.bytes_sent = 0
        self.device = device
        self.rig_send = self.rig_all = None   # impulse all-gather buffers, allocated at the first rigid-coupled substep
        if dist is not None and world > 1 and hasattr(adapter, "share_id_end"):
            adapter.share_id_end(dist)        # every id of the run has a colour entry on every rank

    def _reduce_impulses(self):
        """After a whole transfer: every rank's partial impulse sums to every rank (all-gather), summed in rank order."""
        torch, a = self.torch, self.a
        if self.rig_send is None:
            n = a.rigid_impulse_bytes()
            self.rig_send = torch.empty(n, dtype=torch.uint8, device=self.device)
            self.rig_all = torch.empty(n * self.world, dtype=torch.uint8, device=self.device)
        a.rigid_impulse_pack(self.rig_send)
        self.dist.all_gather(list(self.rig_all.chunk(self.world)), self.rig_send, group=self.group)   # rank r's block r
        a.rigid_impulse_apply(self.rig_all)

    def _exchange(self, send, recv, wait=True):
        """send[0] -> rank-1, send[1] -> rank+1 ; recv[0] <- rank-1, recv[1] <- rank+1.
        wait=False returns the in-flight work handles (the caller overlaps compute, then waits)."""
        d = self.dist
        ops = []
        if self.has_lo:
            ops.append(d.P2POp(d.isend, send[0], self.rank - 1, self.group))
            ops.append(d.P2POp(d.irecv, recv[0], self.rank - 1, self.group))
        if self.has_hi:
            ops.append(d.P2POp(d.isend, send[1], self.rank + 1, self.group))
            ops.append(d.P2POp(d.irecv, recv[1], self.rank + 1, self.group))
        works = []
        if ops:
            works = d.batch_isend_irecv(ops)
            self.bytes_sent += sum(op.tensor.numel() for op in ops[::2])
            if wait:
                for w in works:
                    w.wait()
                works = []
        return works

    def substep(self, n=1):
        a = self.a
        rigid = self.world > 1 and hasattr(a, "rigid_on") and a.rigid_on()
        for _ in range(n):
            a.sort()
            if self.world == 1:
                a.rasterize()
                a.resample()
                continue
            if self.overlap:
                # boundary-layer tiles first; their arenas fly to the neighbours while the interior
                # tiles are rasterized and resampled; the boundary tiles are resampled last
                a.rasterize_part(1)
                if self.has_lo:
                    a.halo_pack(0, self.halo_send[0])
                if self.has_hi:
                    a.halo_pack(1, self.halo_send[1])
                works = self._exchange(self.halo_send, self.halo_recv, wait=False)
                a.rasterize_part(2)
                if rigid:
                    self._reduce_impulses()
                a.resample_part(2)
                for w in works:
                    w.wait()
                if self.has_lo:
                    a.halo_unpack(0, self.halo_recv[0])
                if self.has_hi:
                    a.halo_unpack(1, self.halo_recv[1])
                a.resample_part(1)
                if rigid:
                    self._reduce_impulses()
            else:
                a.rasterize()
                if rigid:
                    self._reduce_impulses()
                if self.has_lo:
                    a.halo_pack(0, self.halo_send[0])
                if self.has_hi:
                    a.halo_pack(1, self.halo_send[1])
                self._exchange(self.halo_send, self.halo_recv)
                if self.has_lo:
                    a.halo_unpack(0, self.halo_recv[0])
                if self.has_hi:
                    a.halo_unpack(1, self.halo_recv[1])
                a.resample()
                if rigid:
                    self._reduce_impulses()
            if self.world > 1:
                if self.has_lo:
                    a.migrate_pack(0, self.mig_send[0])
                if self.has_hi:
                    a.migrate_pack(1, self.mig_send[1])
                self._exchange(self.mig_send, self.mig_recv)
                if self.has_lo:
                    a.migrate_unpack(0, self.mig_recv[0])
                if self.has_hi:
                    a.migrate_unpack(1, self.mig_recv[1])


class SlabEditError(RuntimeError):
    """An edit failed on another rank of the run (the failing rank raises the engine's own error)."""


def _on_all_ranks(call, dist, op):
    """Runs `call` on this rank and reduces its integer result over the ranks with dist.ReduceOp.<op> (dist None: one engine).
    A failure on any rank raises on every rank, after the reduction, so that no rank is left waiting in a later collective."""
    err, value = None, 0
    try:
        value = int(call())
    except Exception as e:  # noqa: BLE001 - re-raised below, after the other ranks have heard of it
        err = e
    if dist is None:
        if err is not None:
            raise err
        return value
    import torch
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    failed = torch.tensor([1 if err is not None else 0], dtype=torch.int64, device=dev)
    total = torch.tensor([value], dtype=torch.int64, device=dev)
    dist.all_reduce(failed, op=dist.ReduceOp.MAX)
    dist.all_reduce(total, op=getattr(dist.ReduceOp, op))
    if err is not None:
        raise err
    if int(failed.item()):
        raise SlabEditError("the edit failed on another rank")
    return int(total.item())


def global_id_end(engine, dist=None):
    """The next free particle id of the run: the maximum of engine.id_end() over the ranks."""
    _refuse_2d(engine)
    return _on_all_ranks(engine.id_end, dist, "MAX")


def share_id_end(engine, dist=None):
    """Raises this rank's id end to the run's (global_id_end) and returns it.  A z-slab rank with rigid coupling keeps the
    particles' colour states by absolute id below its id end, and an immigrant may carry any id of the run: after per-rank
    uploads (set_id_base + upload, seed_lattice) every rank must know the run's id end.  connect_peers and SlabRunner call it."""
    _refuse_2d(engine)
    end = global_id_end(engine, dist)
    z3, z1 = np.zeros((0, 3), np.float32), np.zeros(0, np.float32)
    engine.append_owned(z3, z3, z1, z1, first_id=end)   # no particle: only the id end moves
    return end


def append_particles(engine, batch, first_id, dist=None):
    """Adds a batch of particles to a z-slab run (or to one engine with dist=None) between substeps, keeping every resident
    particle's id and state.  Every rank passes the SAME batch (dict x, v, mass, vol and optionally F, b, ps, group) and the
    same first_id (at least global_id_end); particle k gets id first_id + k on the rank that owns it.  Returns the number
    kept over all ranks (particles outside the domain are dropped, their ids consumed).
    If a rank fails, every rank raises.  A rank whose configured capacity is too small raises MPMB_ERR_CAPACITY and is left
    unchanged, but the other ranks have made their part of the edit: the run is then inconsistent.  Engines created with
    capacity 0 (the default) grow instead and never fail this way."""
    _refuse_2d(engine)
    return _on_all_ranks(lambda: engine.append_owned(batch["x"], batch["v"], batch["mass"], batch["vol"], batch.get("F"), batch.get("b"),
                                                     batch.get("ps"), batch.get("group"), first_id=first_id),
                         dist, "SUM")


def delete_inside_levelset(engine, dist=None):
    """Removes the particles inside the level set (phi < 0) on every rank; returns the number removed over all ranks."""
    _refuse_2d(engine)
    return _on_all_ranks(engine.delete_owned_inside_levelset, dist, "SUM")


def connect_peers(engine, rank, world, dist):
    """Maps the ring neighbours' receive buffers and every rank's rigid impulse mailbox into `engine` with CUDA IPC (one
    process per GPU): afterwards engine.substep(n) runs whole z-slab substeps, halo, migration and the rigid impulse
    reductions included, with no host transport.  Handles travel through torch.distributed once."""
    _refuse_2d(engine)
    share_id_end(engine, dist)
    mine = {(k, f): engine.xchg_ipc_handle(k, f) for k in (0, 1) for f in (0, 1)}
    mine["rigid"] = engine.rigid_mailbox_ipc_handle()
    everyone = [None] * world
    dist.all_gather_object(everyone, mine)
    for r in range(world):   # the rigid impulse mailboxes: every rank's, for the reductions of rigid-coupled substeps
        if r != rank:
            engine.rigid_connect(r, handle=everyone[r]["rigid"])
    for k in (0, 1):
        if rank > 0:
            engine.xchg_connect(k, 0, handle=everyone[rank - 1][(k, 1)])   # my face 0 -> lower neighbour's face-1 buffer
        if rank < world - 1:
            engine.xchg_connect(k, 1, handle=everyone[rank + 1][(k, 0)])   # my face 1 -> upper neighbour's face-0 buffer
    dist.barrier()


def rebalance(engine, rank, world, dist, cuts=None):
    """Re-cuts a z-slab run between substeps (every rank calls it at the same substep boundary): the cuts balance the run's
    particle histogram again (partition_counts of the layer counts summed over the ranks), or are `cuts` ([(z0, z1)] per
    rank) when given, and the particles move to their new owner ranks with their ids and state.  Returns (old_cuts,
    new_cuts, rows_moved over all ranks); unchanged cuts move nothing.

    The bytes go through dist.all_to_all_single on device buffers (NCCL) rather than the ring neighbours' peer mappings: a
    re-cut is rare and may send particles to any rank.  Configured capacities are checked on every rank before any rank
    changes; if one is too small, every rank raises SlabEditError and nothing changes."""
    _refuse_2d(engine)
    import torch
    from .capi import RECORD_BYTES
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    mine = np.asarray(engine.layer_counts(), np.int64)
    hist = torch.as_tensor(mine, device=dev)
    dist.all_reduce(hist)
    ranges = [None] * world
    dist.all_gather_object(ranges, tuple(engine.tile_range()))
    old = [tuple(int(z) for z in r) for r in ranges]
    new = partition_counts(hist.cpu().numpy(), world) if cuts is None else [(int(a), int(b)) for a, b in cuts]
    if new == old:
        return old, new, 0
    flat = [new[0][0]] + [z1 for _, z1 in new]
    z0, z1 = new[rank]
    send_n = np.asarray(engine.recut_pack(flat), np.int64)   # per destination rank
    recv_t = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_to_all_single(recv_t, torch.as_tensor(send_n, device=dev))
    recv_n = recv_t.cpu().numpy()
    n_in = int(recv_n.sum())

    def capacity_check():
        need, cap = int(mine[z0:z1].sum()) + n_in, int(engine.cfg.capacity)
        if cap > 0 and need > cap:
            raise SlabEditError("rank %d: %d particles after the re-cut exceed its configured capacity %d" % (rank, need, cap))
        return int(send_n.sum())

    moved = _on_all_ranks(capacity_check, dist, "SUM")
    send = torch.empty(int(send_n.sum()) * RECORD_BYTES, dtype=torch.uint8, device=dev)
    engine.recut_pack(flat, send)
    recv = torch.empty(n_in * RECORD_BYTES, dtype=torch.uint8, device=dev)
    dist.all_to_all_single(recv, send, [int(c) * RECORD_BYTES for c in recv_n], [int(c) * RECORD_BYTES for c in send_n])
    _on_all_ranks(lambda: engine.recut_apply(z0, z1, recv, n_in) or 0, dist, "SUM")
    return old, new, moved
