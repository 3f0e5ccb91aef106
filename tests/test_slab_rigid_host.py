"""SlabRunner's rigid impulse reductions on CPU: gloo processes at world 2 and 3 and a mock engine.  After each whole transfer
(both parts in the overlap schedule) every rank packs its partial sums, the all-gather hands every rank all partials in rank
order, and the engine applies them before the next stage; the run's id end is shared at set-up."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from taichi_mpm_b200 import slab
from tests.test_slab_host import MockAdapter

NBYTES = 288   # 12 bodies x 6 floats


class RigidMock(MockAdapter):
    def __init__(self, rank):
        super().__init__(rank)
        self.end = 100 * (rank + 1)      # per-rank uploads: rank r's ids end at 100 (r + 1)
        self.gathered = []

    def share_id_end(self, d):
        t = torch.tensor([self.end], dtype=torch.int64)
        d.all_reduce(t, op=d.ReduceOp.MAX)
        self.end = int(t.item())
        self.log.append("ids")

    def rigid_on(self):
        return True

    def rigid_impulse_bytes(self):
        return NBYTES

    def rigid_impulse_pack(self, buf):
        buf.fill_(self.rank + 1 + 10 * len(self.gathered))
        self.log.append("pack")

    def rigid_impulse_apply(self, buf):
        self.gathered.append([int(b[0]) for b in buf.chunk(buf.numel() // NBYTES)] if all(bool((b == b[0]).all()) for b in buf.chunk(buf.numel() // NBYTES)) else None)
        self.log.append("apply")


def _worker(rank, world, port, q, overlap):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    a = RigidMock(rank)
    r = slab.SlabRunner(a, rank, world, torch.device("cpu"), dist=dist, overlap=overlap)
    r.substep(2)
    q.put((rank, a.log, a.gathered, a.end))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("world,overlap", [(2, False), (3, False), (2, True), (3, True)])
def test_impulse_all_gather_choreography_gloo(world, overlap):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, overlap)) for r in range(world)]
    for p in procs:
        p.start()
    out = {}
    for _ in range(world):
        rank, log, gathered, end = q.get(timeout=120)
        out[rank] = (log, gathered, end)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in range(world):
        log, gathered, end = out[rank]
        lo, hi = rank > 0, rank < world - 1
        red = ["pack", "apply"]
        hp = (["hp0"] if lo else []) + (["hp1"] if hi else [])
        hu = (["hu0"] if lo else []) + (["hu1"] if hi else [])
        mig = (["mp0"] if lo else []) + (["mp1"] if hi else []) + (["mu0"] if lo else []) + (["mu1"] if hi else [])
        plain = ["sort", "p2g"] + red + hp + hu + ["g2p"] + red + mig
        # overlap: the P2G reduction after both rasterize parts (before any resample), the G2P one after both resample parts
        step = ["sort", "p2g1"] + hp + ["p2g2"] + red + ["g2p2"] + hu + ["g2p1"] + red + mig
        assert log == ["ids"] + (step if overlap else plain) * 2
        assert end == 100 * world
        # every reduction saw every rank's partial of THAT reduction, in rank order
        assert gathered == [[r + 1 + 10 * k for r in range(world)] for k in range(4)]
