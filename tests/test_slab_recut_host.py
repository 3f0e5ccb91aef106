"""slab.rebalance on CPU: world-size 2, 3 and 8 `gloo` processes, each with a stand-in engine that holds particles as
(id, tile layer) records, check that every record reaches the rank that owns its layer under the new cuts, that every rank
takes the same cuts, and that a configured capacity too small on one rank raises on every rank before any rank applies
(no CUDA here)."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from taichi_mpm_b200 import slab
from taichi_mpm_b200.capi import RECORD_BYTES

N_LAYERS = 40


class _Cfg:
    def __init__(self, capacity):
        self.capacity = capacity


class MockEngine:
    """Stand-in for capi.Engine on a z-slab rank: particle k is the record (id, layer) padded to RECORD_BYTES, kept in
    storage order; recut_pack / recut_apply follow the engine's contract (include/mpmb.h) on the host."""

    def __init__(self, rank, z0, z1, ids, layers, capacity=0):
        self.rank, self.z = rank, (z0, z1)
        self.ids, self.layers = np.asarray(ids, np.int64), np.asarray(layers, np.int64)
        self.cfg = _Cfg(capacity)
        self.applied = []

    def tile_range(self):
        return self.z

    def layer_counts(self):
        return np.bincount(self.layers, minlength=N_LAYERS)

    def _dest(self, flat):
        return np.searchsorted(np.asarray(flat[1:]), self.layers, side="right")

    def recut_pack(self, flat, buf=None):
        dest = self._dest(flat)
        world = len(flat) - 1
        counts = np.array([0 if d == self.rank else int((dest == d).sum()) for d in range(world)], np.int64)
        if buf is not None:
            rec = buf.numpy().view(np.int64).reshape(-1, RECORD_BYTES // 8)
            assert len(rec) == counts.sum()
            o = 0
            for d in range(world):
                if d == self.rank:
                    continue
                sel = np.nonzero(dest == d)[0]
                rec[o:o + len(sel), 0], rec[o:o + len(sel), 1] = self.ids[sel], self.layers[sel]
                o += len(sel)
        return counts

    def recut_apply(self, z0, z1, buf, n_in):
        rec = buf.numpy().view(np.int64).reshape(-1, RECORD_BYTES // 8)
        assert len(rec) == n_in and ((rec[:, 1] >= z0) & (rec[:, 1] < z1)).all()
        stay = (self.layers >= z0) & (self.layers < z1)
        self.ids = np.concatenate([self.ids[stay], rec[:, 0]])
        self.layers = np.concatenate([self.layers[stay], rec[:, 1]])
        self.z = (z0, z1)
        self.applied.append((z0, z1))


def _start(rank, world):
    """The same initial even cuts on every rank; particles crowd the upper half of the domain, so the cuts move."""
    flat = [N_LAYERS * r // world for r in range(world)] + [N_LAYERS]
    rng = np.random.default_rng(3)
    layers = np.concatenate([rng.integers(0, N_LAYERS, 300), rng.integers(N_LAYERS // 2, N_LAYERS, 1500)])
    ids = np.arange(len(layers))
    mine = (layers >= flat[rank]) & (layers < flat[rank + 1])
    return flat, ids[mine], layers[mine], layers


def _worker(rank, world, port, small_cap_rank, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    flat, ids, layers, _ = _start(rank, world)
    e = MockEngine(rank, flat[rank], flat[rank + 1], ids, layers, capacity=len(ids) if rank == small_cap_rank else 0)
    try:
        out = slab.rebalance(e, rank, world, dist)
    except slab.SlabEditError as ex:
        out = "raised: " + str(ex)
    again = slab.rebalance(e, rank, world, dist) if not isinstance(out, str) else None   # balanced already: moves nothing
    q.put((rank, out, again, e.ids, e.layers, e.z, e.applied))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world, small_cap_rank=-1):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, small_cap_rank, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = {}
    for _ in range(world):
        r = q.get(timeout=120)
        out[r[0]] = r[1:]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


@pytest.mark.parametrize("world", [2, 3, 8])
def test_rebalance_sends_every_record_to_its_owner_and_every_rank_takes_the_same_cuts(world):
    out = _run(world)
    flat, _, _, layers = _start(0, world)
    want = slab.partition_counts(np.bincount(layers, minlength=N_LAYERS), world)
    old = [(flat[r], flat[r + 1]) for r in range(world)]
    assert want != old
    moved_want = sum(int(((layers >= a) & (layers < b)).sum() - ((layers >= max(a, c)) & (layers < min(b, d))).sum())
                     for (a, b), (c, d) in zip(old, want))
    ids = []
    for rank in range(world):
        res, again, r_ids, r_layers, z, applied = out[rank]
        assert res == (old, want, moved_want)
        assert again == (want, want, 0) and applied == [want[rank]] and z == want[rank]
        assert ((r_layers >= z[0]) & (r_layers < z[1])).all()
        ids.append(r_ids)
    ids = np.concatenate(ids)
    assert np.array_equal(np.sort(ids), np.arange(len(layers)))   # every particle on exactly one rank


@pytest.mark.parametrize("world", [2, 3])
def test_capacity_failure_on_one_rank_raises_on_every_rank_before_any_apply(world):
    out = _run(world, small_cap_rank=0)   # rank 0 takes more layers of the crowded half
    for rank in range(world):
        res, again, r_ids, _, z, applied = out[rank]
        assert isinstance(res, str) and "raised" in res
        if rank == 0:
            assert "configured capacity" in res
        assert applied == [] and again is None
        flat, ids, _, _ = _start(rank, world)
        assert z == (flat[rank], flat[rank + 1]) and np.array_equal(r_ids, ids)
