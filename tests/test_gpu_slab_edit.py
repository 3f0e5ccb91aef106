"""Edits of the resident particle set on z-slab ranks (mpmb_append_owned_particles, mpmb_delete_owned_inside_levelset,
mpmb_id_end and the slab.py helpers around them): every rank receives the same batch, keeps the particles it owns and
numbers them first_id + k, so a slab run that appends and deletes between substeps ends where one engine making the same
edits with mpmb_append_particles / mpmb_delete_inside_levelset ends.  Runs on the SIMT emulator too
(tests/test_slab_edit_simt.py)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

from taichi_mpm_b200 import capi, scenes, slab
from tests import common as T
from tests.test_gpu_slab import SIMT, _HostBuf, _long_scene, _scene

pytestmark = pytest.mark.gpu

KEYS = ("x", "v", "mass", "vol", "F", "b", "ps", "group")
OUT = ("id", "x", "v", "F", "b", "mass", "vol", "ps", "group")
TOL = (("x", 2e-6), ("v", 5e-4), ("F", 5e-5), ("ps", 1e-5))   # the slab tolerances of tests/test_gpu_slab.py
MIG_CAP = 64   # small migration buffers: the first append outgrows the rows reserved at upload (n + n/4 + 16 * MIG_CAP)


def _sand(x, seed):
    """Sand particles at x (the scene's lattice mass and volume) moving along +z where x < 0.5 and along -z elsewhere."""
    vol = np.full(len(x), np.float32(1.0 / 32) ** 3 / 8, np.float32)
    st = scenes.make_state(x.astype(np.float32), vol * 400, vol, scenes.MAT_SAND)
    rng = np.random.default_rng(seed)
    vz = np.where(x[:, 0] < 0.5, 2.5, -2.5)
    st["v"] = np.stack([0.3 * rng.normal(size=len(x)), 0.3 * rng.normal(size=len(x)), vz + 0.2 * rng.normal(size=len(x))], 1).astype(np.float32)
    return {k: np.ascontiguousarray(st[k]) for k in KEYS}


def _batch(cuts, z_cells, lattice_cells, seed):
    """A batch above the block that spans the slab cuts inside z_cells: a jittered lattice of lattice_cells[0] x
    lattice_cells[1] cells in x, y, plus, at every cut c (tile layer), particles whose base node is the last node layer of
    the lower slab (z = 4c + 0.48 cells, moving up) and the first node layer of the upper slab (4c + 0.52, moving down):
    they cross the cut within a few substeps."""
    dx = 1.0 / 32
    lx, ly = lattice_cells
    x, _, _ = scenes.lattice_block(32, (11, 18, z_cells[0]), (11 + lx, 18 + ly, z_cells[1]), jitter=0.2, seed=seed)
    rng = np.random.default_rng(seed)
    edge = []
    for z0, _ in cuts[1:]:
        for dz, xs in ((0.48, 12.0), (0.52, 19.5)):   # x < 16 moves +z, x > 16 moves -z (_sand)
            k = 12
            X = np.stack([xs + rng.uniform(0, 1, k), 18.0 + ly + 0.3 + rng.uniform(0, 0.6, k), np.full(k, 4 * z0 + dz)], 1)
            edge.append(X * dx)
    x = np.concatenate([x] + edge).astype(np.float32)
    return _sand(x, seed + 1)


class _Slabs:
    """`world` z-slab engines of one scene in one process on one device.  peer=True: the exchange goes through the
    engine's peer-memory path with interleaved stages; peer=False (world 2): the host moves the buffers (EngineAdapter)."""

    def __init__(self, scene, st, world, peer):
        if not SIMT:
            import torch
            self.torch = torch
        self.scene, self.world, self.peer = scene, world, peer
        tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
        self.cuts = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)
        counts = [int(((tz >= a) & (tz < b)).sum()) for a, b in self.cuts]
        assert min(counts) > 0
        self.order = np.concatenate([np.nonzero((tz >= a) & (tz < b))[0] for a, b in self.cuts])
        self.n0 = len(st["x"])
        self.eng = []
        for rank, (z0, z1) in enumerate(self.cuts):
            e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], 1, True, device=0, rank=rank, world=world,
                            tile_z0=z0, tile_z1=z1, migrate_capacity=MIG_CAP, halo_capacity=64)
            if not peer and not SIMT:
                e.set_stream(self.torch.cuda.current_stream().cuda_stream)
            e.set_material(0, int(scene["mat_kind"][0]), scene["mat_params"][0])
            e.set_planes(scene["planes"], scene["friction"])
            e.set_id_base(sum(counts[:rank]))
            mine = np.nonzero((tz >= z0) & (tz < z1))[0]
            e.upload(*(st[k][mine] for k in KEYS))
            self.eng.append(e)
        if peer:
            for r in range(world - 1):
                for k in (0, 1):
                    self.eng[r].xchg_connect(k, 1, ptr=self.eng[r + 1].xchg_buffer(k, 0))
                    self.eng[r + 1].xchg_connect(k, 0, ptr=self.eng[r].xchg_buffer(k, 1))
            self.faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < world] for r in range(world)]
        else:
            assert world == 2
            dev = None if SIMT else self.torch.device("cuda", 0)
            mk = (lambda n: _HostBuf(max(int(n), 16))) if SIMT else (lambda n: self.torch.zeros(max(int(n), 16), dtype=self.torch.uint8, device=dev))
            self.ad = [slab.EngineAdapter(e) for e in self.eng]
            self.bufs = [dict(halo=[mk(e.halo_bytes()), mk(e.halo_bytes())], mig=[mk(e.migrate_bytes()), mk(e.migrate_bytes())]) for e in self.eng]

    def step(self, n):
        for _ in range(n):
            if self.peer:   # one stream, one process: every wait finds its flag already published
                for e in self.eng:
                    e.sort_particles_and_populate_grid(); e.rasterize()
                for f_e in (lambda e, f: e.halo_send(f), lambda e, f: e.halo_recv(f)):
                    for r, e in enumerate(self.eng):
                        for f in self.faces[r]:
                            f_e(e, f)
                for e in self.eng:
                    e.resample()
                for f_e in (lambda e, f: e.migrate_send(f), lambda e, f: e.migrate_recv(f)):
                    for r, e in enumerate(self.eng):
                        for f in self.faces[r]:
                            f_e(e, f)
            else:
                (a0, a1), (b0, b1) = self.ad, self.bufs
                for a in self.ad:
                    a.sort(); a.rasterize_part(1)
                a0.halo_pack(1, b0["halo"][1]); a1.halo_pack(0, b1["halo"][0])
                for a in self.ad:
                    a.rasterize_part(2); a.resample_part(2)
                a1.halo_unpack(0, b0["halo"][1]); a0.halo_unpack(1, b1["halo"][0])
                for a in self.ad:
                    a.resample_part(1)
                a0.migrate_pack(1, b0["mig"][1]); a1.migrate_pack(0, b1["mig"][0])
                a1.migrate_unpack(0, b0["mig"][1]); a0.migrate_unpack(1, b1["mig"][0])
        if not SIMT and not self.peer:
            self.torch.cuda.synchronize()

    def append(self, batch):
        """Every rank gets the batch and the run's next free id; returns (first_id, kept per rank)."""
        first = max(slab.global_id_end(e) for e in self.eng)
        return first, [slab.append_particles(e, batch, first) for e in self.eng]

    def delete(self):
        return [slab.delete_inside_levelset(e) for e in self.eng]

    def set_planes(self, planes):
        for e in self.eng:
            e.set_planes(planes, self.scene["friction"])

    def parts(self):
        """download() of every rank, with gid = the particle's id in the one-engine run (uploaded ids map through the
        partition order, appended ids are the same on both sides)."""
        out = []
        for e in self.eng:
            g = e.download()
            ids = g["id"].astype(np.int64)
            g["gid"] = np.where(ids < self.n0, self.order[np.minimum(ids, self.n0 - 1)], ids)
            out.append(g)
        return out

    def close(self):
        for e in self.eng:
            e.close()


def _assert_match(parts, ref):
    gid = np.concatenate([p["gid"] for p in parts])
    assert len(np.unique(gid)) == len(gid), "an id lives on two ranks"
    o = np.argsort(gid)
    assert np.array_equal(gid[o], ref["id"].astype(np.int64))
    for k, tol in TOL:
        got = np.concatenate([p[k] for p in parts])[o]
        scale = max(np.abs(ref[k]).max(), 1e-30) if k == "v" else 1.0
        assert np.abs(got - ref[k]).max() <= tol * scale, k


def _owner(parts):
    return {int(g): r for r, p in enumerate(parts) for g in p["gid"]}


def _cut_plane(x, dx, frac):
    """A plane tilted along z, through every slab, with `frac` of the particles below it and none within 1e-4 grid units
    of it: slab and single-engine positions may differ by the slab tolerance (6e-5 grid units here), the decision must not."""
    n = np.array([0.0, 1.0, 0.12]) / np.linalg.norm([0.0, 1.0, 0.12])
    n32 = n.astype(np.float32)
    s = np.sort((x.astype(np.float64) / dx) @ n32.astype(np.float64))
    mid = 0.5 * (s[1:] + s[:-1])
    ok = np.nonzero(s[1:] - s[:-1] > 2e-4)[0]
    d = mid[ok[np.argmin(np.abs(mid[ok] - np.quantile(s, frac)))]]
    return np.array([[n32[0], n32[1], n32[2], -d]], np.float32)


def _edit_run(scene, st, world, peer, z_cells, lattice_cells, steps=(6, 6, 6, 4)):
    """k substeps; append a batch across the cuts (it outgrows the reserved rows); k substeps; delete below a tilted plane;
    k substeps; a second append; k substeps — on `world` slabs and on one engine with the legacy calls."""
    S = _Slabs(scene, st, world, peer)
    ref = T.make_engine(scene, st)
    A = _batch(S.cuts, z_cells, lattice_cells, seed=11)
    B = _batch(S.cuts, z_cells, (3, 1), seed=12)
    S.step(steps[0]); ref.substep(steps[0])

    n_before = ref.num_particles()
    first, kept = S.append(A)
    assert first == ref.append(*(A[k] for k in KEYS)) == len(st["x"])
    assert sum(kept) == ref.num_particles() - n_before == len(A["x"]) and min(kept) > 0
    parts = S.parts()
    _assert_match(parts, ref.download())
    at_append = _owner(parts)
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    for (z0, z1), p in zip(S.cuts, parts):   # more live rows than upload reserved: every rank grew, keeping rx / tx
        n_up = int(((tz >= z0) & (tz < z1)).sum())
        assert len(p["gid"]) > n_up + n_up // 4 + 16 * MIG_CAP
    S.step(steps[1]); ref.substep(steps[1])

    cut = _cut_plane(ref.download()["x"], scene["dx"], 0.3)
    S.set_planes(cut); ref.set_planes(cut, scene["friction"])
    deleted = S.delete()
    n_ref = ref.delete_inside_levelset()
    assert sum(deleted) == n_ref > 0 and sum(1 for d in deleted if d > 0) >= 2
    _assert_match(S.parts(), ref.download())
    S.set_planes(scene["planes"]); ref.set_planes(scene["planes"], scene["friction"])
    S.step(steps[2]); ref.substep(steps[2])

    first2, kept2 = S.append(B)
    assert first2 == ref.append(*(B[k] for k in KEYS)) == first + len(A["x"])
    S.step(steps[3]); ref.substep(steps[3])
    parts = S.parts()
    _assert_match(parts, ref.download())
    assert sum(kept2) == len(B["x"])
    now = _owner(parts)
    moved = [(at_append[g], now[g]) for g in range(first, first + len(A["x"])) if g in now and now[g] != at_append[g]]
    assert any(b > a for a, b in moved) and any(b < a for a, b in moved), "appended particles did not migrate both ways"
    assert max(slab.global_id_end(e) for e in S.eng) == first2 + len(B["x"])
    S.close(); ref.close()


def test_two_slabs_host_moved_buffers_edit_like_one_engine():
    scene, st = _scene()
    _edit_run(scene, st, 2, peer=False, z_cells=(14, 50), lattice_cells=(10, 4))


def test_four_slabs_peer_memory_edit_like_one_engine():
    scene, st = _scene()
    _edit_run(scene, st, 4, peer=True, z_cells=(14, 50), lattice_cells=(10, 5))


def test_eight_slabs_peer_memory_edit_like_one_engine():
    scene, st = _long_scene()
    _edit_run(scene, st, 8, peer=True, z_cells=(14, 114), lattice_cells=(10, 3), steps=(4, 4, 4, 4))


def test_append_owned_on_one_engine_equals_append_bit_for_bit():
    scene, st = _scene()
    A = _batch([(0, 8), (8, 17)], (14, 50), (4, 2), seed=21)
    A["x"][:3] = np.array([[-0.05, 0.5, 0.5], [0.5, 0.5, 2.5], [0.5, -0.05, 0.5]], np.float32)   # dropped, ids consumed
    outs = []
    for owned in (False, True):
        e = T.make_engine(scene, st)
        e.substep(5)
        if owned:
            assert e.append_owned(*(A[k] for k in KEYS), first_id=e.id_end()) == len(A["x"]) - 3
        else:
            assert e.append(*(A[k] for k in KEYS)) == len(st["x"])
        assert e.id_end() == len(st["x"]) + len(A["x"])
        after = e.download()
        assert e.append(*(A[k][3:] for k in KEYS)) == len(st["x"]) + len(A["x"])   # the legacy call continues after both
        e.substep(7)
        outs.append((after, e.download()))
        e.close()
    for a, b in zip(outs[0], outs[1]):
        assert len(a["id"]) == len(b["id"])
        for k in OUT:
            assert np.array_equal(a[k], b[k]), k


def test_append_after_seeding_slab_ranks_takes_ids_past_the_whole_lattice():
    scene, st = _scene()
    lo, hi = (10, 9, 12), (22, 17, 52)
    lattice = 8 * int(np.prod(np.subtract(hi, lo)))
    vol = np.float32(scene["dx"]) ** 3 / 8
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    cuts = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), 3)
    eng = []
    for rank, (z0, z1) in enumerate(cuts):
        e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], rank=rank, world=3, tile_z0=z0, tile_z1=z1, migrate_capacity=4096)
        e.set_material(0, int(scene["mat_kind"][0]), scene["mat_params"][0])
        assert 0 < e.seed_lattice(lo, hi, vol, vol * 400, jitter=0.2, seed=4) < lattice
        assert e.id_end() == lattice
        eng.append(e)
    first = max(slab.global_id_end(e) for e in eng)
    assert first == lattice
    A = _batch(cuts, (14, 50), (4, 2), seed=31)
    assert sum(slab.append_particles(e, A, first) for e in eng) == len(A["x"])
    ids = np.concatenate([e.download()["id"].astype(np.int64) for e in eng])
    assert len(np.unique(ids)) == len(ids)
    assert np.array_equal(np.sort(ids[ids >= lattice]), np.arange(lattice, lattice + len(A["x"])))
    assert (ids[ids < lattice] >= 0).all()
    for e in eng:
        e.close()


def _snapshot(e):
    return e.num_particles(), e.id_end(), e.download()


def _assert_unchanged(e, snap):
    n, end, d = _snapshot(e)
    assert n == snap[0] and end == snap[1]
    assert len(d["id"]) == len(snap[2]["id"])
    for k in OUT:
        assert np.array_equal(d[k], snap[2][k]), k


def test_errors_change_nothing():
    scene, st = _scene()
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    cuts = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), 2)
    mine = np.nonzero(tz < cuts[0][1])[0]
    A = _batch(cuts, (14, 50), (4, 2), seed=41)
    add = lambda e, first, **kw: e.append_owned(*(A[k] for k in KEYS), first_id=first, **kw)
    for capacity in (0, len(mine) + 10):
        e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], rank=0, world=2, tile_z0=cuts[0][0], tile_z1=cuts[0][1],
                        migrate_capacity=4096, capacity=capacity)
        e.set_material(0, int(scene["mat_kind"][0]), scene["mat_params"][0])
        e.set_planes(scene["planes"], scene["friction"])
        e.set_id_base(100)
        e.upload(*(st[k][mine] for k in KEYS))
        end = e.id_end()
        assert end == 100 + len(mine)
        snap = _snapshot(e)
        cases = [(lambda: add(e, end - 1), -1),                                          # first_id below the id end
                 (lambda: add(e, 2 ** 28 - len(A["x"]) + 1), -3),                         # ids past 2^28
                 (lambda: e.append_owned(A["x"], None, A["mass"], A["vol"], first_id=end), -1),
                 (lambda: e.append_owned(A["x"], A["v"], A["mass"], None, first_id=end), -1)]
        if capacity:
            cases.append((lambda: add(e, end), -3))                                      # the configured capacity is too small
        for call, code in cases:
            with pytest.raises(capi.MpmbError) as ex:
                call()
            assert ex.value.code == code
            _assert_unchanged(e, snap)
        n = C.c_int64(0)
        x, v, m, vol = (np.ascontiguousarray(A[k]) for k in ("x", "v", "mass", "vol"))
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert e.L.mpmb_append_owned_particles(e.h, C.c_int64(len(x)), p(x), None, None, None, p(m), p(vol), None, None, C.c_int64(end), C.byref(n)) == -1
        assert e.L.mpmb_append_owned_particles(e.h, C.c_int64(len(x)), p(x), p(v), None, None, p(m), p(vol), None, None, C.c_int64(end), None) == -1
        assert e.L.mpmb_delete_owned_inside_levelset(e.h, None) == -1 and e.L.mpmb_id_end(e.h, None) == -1
        _assert_unchanged(e, snap)
        e.sort_particles_and_populate_grid()                                             # inside a substep
        for call in (lambda: add(e, end), e.delete_owned_inside_levelset):
            with pytest.raises(capi.MpmbError) as ex:
                call()
            assert ex.value.code == -4
        e.rasterize_part(1); e.rasterize_part(2); e.resample_part(2); e.resample_part(1)
        if capacity == 0:
            assert add(e, end + 5) > 0 and e.id_end() == end + 5 + len(A["x"])          # nothing was consumed by the refusals
        e.close()


def test_legacy_edits_still_refuse_slab_ranks():
    scene, st = _scene()
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], rank=1, world=2, tile_z0=4, tile_z1=slab.tile_layers(64), migrate_capacity=4096)
    with pytest.raises(capi.MpmbError) as ex:
        e.append(st["x"][:4], st["v"][:4], st["mass"][:4], st["vol"][:4])
    assert ex.value.code == -4
    e.close()


# ---- two GPUs: one process per rank, an append that outgrows the rows on both ranks, then whole substeps

def _spawn_worker(rank, world, port, transport, out_path):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    scene, st = _scene()
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    cuts = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)
    z0, z1 = cuts[rank]
    counts = [int(((tz >= a) & (tz < b)).sum()) for a, b in cuts]
    mine = np.nonzero((tz >= z0) & (tz < z1))[0]
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], 1, True, device=rank, rank=rank, world=world, tile_z0=z0, tile_z1=z1,
                    migrate_capacity=MIG_CAP, halo_capacity=64)
    e.set_stream(torch.cuda.current_stream().cuda_stream)
    e.set_material(0, int(scene["mat_kind"][0]), scene["mat_params"][0])
    e.set_planes(scene["planes"], scene["friction"])
    e.set_id_base(sum(counts[:rank]))
    e.upload(*(st[k][mine] for k in KEYS))
    if transport == "peer":
        slab.connect_peers(e, rank, world, dist)
        run = e.substep
    else:
        r = slab.SlabRunner(slab.EngineAdapter(e), rank, world, torch.device("cuda", rank), dist=dist)
        run = r.substep
    run(6)
    A = _batch(cuts, (14, 50), (10, 4), seed=11)
    first = slab.global_id_end(e, dist)
    before = e.num_particles()
    total = slab.append_particles(e, A, first, dist)
    kept = e.num_particles() - before
    run(10)
    torch.cuda.synchronize()
    e.synchronize()
    got = e.download()
    ids = got["id"].astype(np.int64)
    order = np.concatenate([np.nonzero((tz >= a) & (tz < b))[0] for a, b in cuts])
    got["gid"] = np.where(ids < len(st["x"]), order[np.minimum(ids, len(st["x"]) - 1)], ids)
    np.savez(out_path % rank, **got, first=first, total=total, kept=kept, before=before, n_up=len(mine))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.needs_cuda
@pytest.mark.parametrize("transport", ["nccl", "peer"])
def test_two_ranks_append_with_growth_then_whole_substeps(tmp_path, transport):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out_path = str(tmp_path / "rank%d.npz")
    mp.spawn(_spawn_worker, args=(2, _free_port(), transport, out_path), nprocs=2, join=True)
    scene, st = _scene()
    A = _batch(slab.slab_partition(slab.base_tile_z(st["x"][:, 2], scene["dx"]), slab.tile_layers(scene["res"][2]), 2), (14, 50), (10, 4), seed=11)
    ref = T.make_engine(scene, st)
    ref.substep(6)
    assert ref.append(*(A[k] for k in KEYS)) == len(st["x"])
    ref.substep(10)
    want = ref.download()
    ref.close()
    parts = [dict(np.load(out_path % r)) for r in range(2)]
    for p in parts:
        assert int(p["first"]) == len(st["x"]) and int(p["total"]) == len(A["x"])
        n_up = int(p["n_up"])                                           # more rows than upload reserved: the rank grew
        assert int(p["before"]) + int(p["kept"]) > n_up + n_up // 4 + 16 * MIG_CAP
    _assert_match(parts, want)
