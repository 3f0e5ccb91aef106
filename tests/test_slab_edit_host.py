"""The edit helpers of taichi_mpm_b200/slab.py (global_id_end, append_particles, delete_inside_levelset) on CPU: world-size
2 and 3 `gloo` processes, each with a stand-in engine, check what every rank hands its engine and what every rank gets
back (no CUDA here)."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from taichi_mpm_b200 import slab


class MockEngine:
    """Stand-in for capi.Engine: records the edit calls; rank r keeps r + 1 particles of a batch, deletes 10 * (r + 1) and
    reports an id end of 100 * (r + 1).  `fail` makes one call raise on this rank."""

    def __init__(self, rank, fail=None):
        self.rank, self.fail, self.calls = rank, fail, []

    def _maybe_fail(self, what):
        if self.fail == what:
            raise RuntimeError("engine failure on rank %d" % self.rank)

    def id_end(self):
        self._maybe_fail("id_end")
        return 100 * (self.rank + 1)

    def append_owned(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None, *, first_id):
        self._maybe_fail("append")
        self.calls.append(("append", np.asarray(x).tobytes(), np.asarray(v).tobytes(), scalar is not None, first_id))
        return self.rank + 1

    def delete_owned_inside_levelset(self):
        self._maybe_fail("delete")
        return 10 * (self.rank + 1)


def _batch():
    rng = np.random.default_rng(7)
    n = 5
    return dict(x=rng.random((n, 3), np.float32), v=rng.random((n, 3), np.float32), mass=np.ones(n, np.float32), vol=np.ones(n, np.float32),
                ps=np.zeros(n, np.float32))


def _worker(rank, world, port, fail_rank, fail_what, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    e = MockEngine(rank, fail_what if rank == fail_rank else None)
    out = {}
    for name, call in (("id_end", lambda: slab.global_id_end(e, dist)),
                       ("append", lambda: slab.append_particles(e, _batch(), 1000, dist)),
                       ("delete", lambda: slab.delete_inside_levelset(e, dist))):
        try:
            out[name] = call()
        except slab.SlabEditError:
            out[name] = "other rank failed"
        except RuntimeError as ex:
            out[name] = "raised: " + str(ex)
    q.put((rank, out, e.calls))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world, fail_rank=-1, fail_what=None):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, fail_rank, fail_what, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = {}
    for _ in range(world):
        rank, res, calls = q.get(timeout=120)
        out[rank] = (res, calls)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_helpers_reduce_over_the_ranks_and_hand_every_rank_the_same_batch(world):
    out = _run(world)
    b = _batch()
    for rank in range(world):
        res, calls = out[rank]
        assert res["id_end"] == 100 * world                                    # the maximum
        assert res["append"] == sum(r + 1 for r in range(world))               # totals are sums
        assert res["delete"] == sum(10 * (r + 1) for r in range(world))
        assert calls == [("append", b["x"].tobytes(), b["v"].tobytes(), True, 1000)]   # the same batch and first_id everywhere


@pytest.mark.parametrize("world,fail_what", [(2, "append"), (3, "id_end"), (3, "delete")])
def test_one_ranks_failure_raises_on_every_rank(world, fail_what):
    out = _run(world, fail_rank=world - 1, fail_what=fail_what)
    for rank in range(world):
        res, _ = out[rank]
        want = "raised: engine failure on rank %d" % rank if rank == world - 1 else "other rank failed"
        assert res[fail_what] == want
        for name in {"id_end", "append", "delete"} - {fail_what}:              # the ranks stay in step for the next collective
            assert not isinstance(res[name], str)


def test_helpers_act_on_one_engine_without_dist():
    e = MockEngine(1)
    assert slab.global_id_end(e) == 200 and slab.append_particles(e, _batch(), 300) == 2 and slab.delete_inside_levelset(e) == 20
    e = MockEngine(0, fail="append")
    with pytest.raises(RuntimeError):
        slab.append_particles(e, _batch(), 0)
