"""Re-cut of z-slab runs (mpmb_layer_counts, mpmb_recut_pack, mpmb_recut_apply and slab.rebalance): after the set has
drifted and an append has crowded one slab, the cuts move to the balanced ones and every particle moves to its new owner
rank with its id and state bit for bit; the run then goes on like one engine that never re-cut.  Runs on the SIMT
emulator too (tests/test_slab_recut_simt.py)."""
import os

import numpy as np
import pytest

from taichi_mpm_b200 import capi, scenes, slab
from tests import common as T
from tests.test_gpu_slab import SIMT, _long_scene, _scene
from tests.test_gpu_slab_edit import KEYS, MIG_CAP, OUT, _assert_match, _assert_unchanged, _cut_plane, _free_port, _owner, _sand, _Slabs, _snapshot

pytestmark = pytest.mark.gpu
RB = capi.RECORD_BYTES


class _HostBytes:
    """numpy-backed stand-in for a torch CUDA byte tensor (emulator runs: device memory is host memory)"""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a, np.uint8)

    def data_ptr(self):
        return self.a.ctypes.data

    def numel(self):
        return self.a.size

    def element_size(self):
        return 1


def _buf(nbytes):
    if SIMT:
        return _HostBytes(np.zeros(nbytes, np.uint8))
    import torch
    return torch.empty(nbytes, dtype=torch.uint8, device="cuda")


def _cat(pieces):
    if SIMT:
        return _HostBytes(np.concatenate([p.a for p in pieces]) if pieces else np.zeros(0, np.uint8))
    import torch
    return torch.cat(pieces) if pieces else _buf(0)


def _piece(b, lo, hi):
    return _HostBytes(b.a[lo:hi]) if SIMT else b[lo:hi]


def _recut(S, cuts=None):
    """slab.rebalance's choreography for the engines of one process: the summed layer histogram, the balanced cuts (or
    `cuts`), every rank's pack, every rank handed what the others packed for it (in source rank order), every rank's apply.
    Returns (histogram, new cuts, rows moved)."""
    hist = sum(e.layer_counts() for e in S.eng)
    new = slab.partition_counts(hist, S.world) if cuts is None else [tuple(c) for c in cuts]
    flat = [new[0][0]] + [z1 for _, z1 in new]
    packs = []
    for e in S.eng:
        counts = e.recut_pack(flat)
        b = _buf(int(counts.sum()) * RB)
        assert np.array_equal(e.recut_pack(flat, b), counts)
        packs.append((counts, b))
    for r, e in enumerate(S.eng):
        pieces = []
        for counts, b in packs:
            lo = int(counts[:r].sum())
            if counts[r]:
                pieces.append(_piece(b, lo * RB, (lo + int(counts[r])) * RB))
        n_in = sum(int(c[r]) for c, _ in packs)
        e.recut_apply(new[r][0], new[r][1], _cat(pieces), n_in)
        assert e.tile_range() == new[r]
    S.cuts = new
    return hist, new, sum(int(c.sum()) for c, _ in packs)


def _union(S):
    """Every rank's download, concatenated and ordered by id; and the rank of every particle."""
    parts = [e.download() for e in S.eng]
    d = {k: np.concatenate([p[k] for p in parts]) for k in OUT}
    rank = np.concatenate([np.full(len(p["id"]), r) for r, p in enumerate(parts)])
    o = np.argsort(d["id"], kind="stable")
    return {k: v[o] for k, v in d.items()}, rank[o], parts


def _crowd(S, scene, seed):
    """An append into the lowest slab only: a block of sand beside the column, every base node below the first cut."""
    z1 = S.cuts[0][1]
    x, _, _ = scenes.lattice_block(32, (11, 18, 14), (21, 28, 4 * z1 - 1), jitter=0.2, seed=seed)
    assert (slab.base_tile_z(x[:, 2], scene["dx"]) < z1).all()
    return _sand(x, seed + 1)


def _drifted(scene, st, world, peer, steps=6, seed=51):
    """Slabs and one engine, `steps` substeps of the ±z flow, an append into slab 0, `steps` more."""
    S = _Slabs(scene, st, world, peer)
    ref = T.make_engine(scene, st)
    S.step(steps); ref.substep(steps)
    A = _crowd(S, scene, seed)
    first, kept = S.append(A)
    assert ref.append(*(A[k] for k in KEYS)) == first and kept[0] == len(A["x"]) == sum(kept)
    S.step(steps); ref.substep(steps)
    return S, ref


def _recut_exact(S, scene):
    before, _, _ = _union(S)
    hist, new, moved = _recut(S)
    assert np.array_equal(hist, slab.layer_histogram(slab.base_tile_z(before["x"][:, 2], scene["dx"]), len(hist)))
    after, rank, parts = _union(S)
    assert len(np.unique(after["id"])) == len(after["id"]), "an id lives on two ranks"
    assert len(after["id"]) == len(before["id"])
    for k in OUT:
        assert np.array_equal(after[k].view(np.uint8), before[k].view(np.uint8)), k   # bit for bit
    tz = slab.base_tile_z(after["x"][:, 2], scene["dx"])
    for r, (z0, z1) in enumerate(new):
        assert ((tz[rank == r] >= z0) & (tz[rank == r] < z1)).all()
        assert len(parts[r]["id"]) == int(hist[z0:z1].sum())
    return new, moved


@pytest.mark.parametrize("world,peer", [(2, False), (4, True), (8, True)])
def test_recut_is_exact_and_the_run_goes_on_like_one_engine(world, peer):
    scene, st = _long_scene() if world == 8 else _scene()
    S, ref = _drifted(scene, st, world, peer)
    old = list(S.cuts)
    new, moved = _recut_exact(S, scene)
    assert new != old and moved > 0
    at_cut = _owner(S.parts())
    steps = 8
    S.step(steps); ref.substep(steps)
    parts = S.parts()
    _assert_match(parts, ref.download())
    assert sum(len(p["id"]) for p in parts) == ref.num_particles()
    now = _owner(parts)
    moved = [(at_cut[g], now[g]) for g in at_cut if g in now and now[g] != at_cut[g]]
    assert any(b > a for a, b in moved) and any(b < a for a, b in moved), "no migration both ways after the re-cut"
    S.close(); ref.close()


def test_recut_is_deterministic():
    """The pack and the apply add no order of their own: the same state re-cut twice leaves the same rows in the same storage
    order on every rank, and the same particles a substep later.  (The state is taken before any migration: the order in
    which a migration appends its arrivals is not fixed.)"""
    scene, st = _scene()
    runs = []
    for _ in range(2):
        S = _Slabs(scene, st, 4, True)
        S.append(_crowd(S, scene, 51))
        old = list(S.cuts)
        _recut(S)
        assert S.cuts != old
        rows = [e.download(sort_by_id=False) for e in S.eng]
        S.step(1)
        runs.append((rows, [e.download() for e in S.eng]))
        S.close()
    for a, b in zip(runs[0][0] + runs[0][1], runs[1][0] + runs[1][1]):
        for k in OUT:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


def test_unchanged_cuts_pack_nothing_and_change_nothing():
    scene, st = _scene()
    S, ref = _drifted(scene, st, 4, True, steps=3)
    flat = [S.cuts[0][0]] + [z1 for _, z1 in S.cuts]
    snaps = [_snapshot(e) for e in S.eng]
    for e, snap in zip(S.eng, snaps):
        b = _buf(16 * RB)
        assert not e.recut_pack(flat).any() and not e.recut_pack(flat, b).any()
        _assert_unchanged(e, snap)   # the pack is read-only
    S.close(); ref.close()


@pytest.mark.parametrize("shape", ["one_rank_takes_most", "rank_ends_empty"])
def test_extreme_cuts_then_substeps_like_one_engine(shape):
    """One rank grows from a few layers to most of the domain (its tile arrays grow), or a rank is left with no particles."""
    scene, st = _scene()
    S, ref = _drifted(scene, st, 4, True, steps=3)
    old = list(S.cuts)
    n = slab.tile_layers(scene["res"][2])
    cuts = [(0, n - 3), (n - 3, n - 2), (n - 2, n - 1), (n - 1, n)] if shape == "one_rank_takes_most" else [(0, 3), (3, 8), (8, 10), (10, n)]
    _recut_exact_given(S, scene, cuts)
    counts = [e.num_particles() for e in S.eng]
    if shape == "one_rank_takes_most":
        assert counts[0] == sum(counts) and S.cuts[0][1] - S.cuts[0][0] > 2 * (old[0][1] - old[0][0])
    else:
        assert counts[0] == 0 and min(counts[1:]) > 0
    S.step(6); ref.substep(6)
    _assert_match(S.parts(), ref.download())
    _recut(S)   # and back to balanced cuts
    S.step(4); ref.substep(4)
    _assert_match(S.parts(), ref.download())
    S.close(); ref.close()


def _recut_exact_given(S, scene, cuts):
    before, _, _ = _union(S)
    _recut(S, cuts)
    after, rank, _ = _union(S)
    for k in OUT:
        assert np.array_equal(after[k].view(np.uint8), before[k].view(np.uint8)), k
    tz = slab.base_tile_z(after["x"][:, 2], scene["dx"])
    for r, (z0, z1) in enumerate(cuts):
        assert ((tz[rank == r] >= z0) & (tz[rank == r] < z1)).all()


def test_append_and_delete_after_a_recut_like_one_engine():
    scene, st = _scene()
    S, ref = _drifted(scene, st, 2, False)
    _recut(S)
    S.step(3); ref.substep(3)
    B = _crowd(S, scene, 61)
    first, kept = S.append(B)
    assert ref.append(*(B[k] for k in KEYS)) == first and sum(kept) == len(B["x"])
    plane = _cut_plane(ref.download()["x"], scene["dx"], 0.3)
    S.set_planes(plane); ref.set_planes(plane, scene["friction"])
    deleted = S.delete()
    assert sum(deleted) == ref.delete_inside_levelset() > 0
    S.set_planes(scene["planes"]); ref.set_planes(scene["planes"], scene["friction"])
    S.step(4); ref.substep(4)
    _assert_match(S.parts(), ref.download())
    assert max(slab.global_id_end(e) for e in S.eng) == first + len(B["x"])
    S.close(); ref.close()


def test_errors_change_nothing():
    scene, st = _scene()
    n = slab.tile_layers(scene["res"][2])
    one = T.make_engine(scene, st)
    for call in (one.layer_counts, lambda: one.recut_pack([0, n]), lambda: one.recut_apply(0, n, None, 0)):
        with pytest.raises(capi.MpmbError) as ex:
            call()
        assert ex.value.code == -4
    one.close()
    S, ref = _drifted(scene, st, 2, False, steps=3)
    e0, e1 = S.eng
    snaps = [_snapshot(e) for e in S.eng]
    flat = [0, S.cuts[0][1] + 2, n]
    cases = [(lambda: e0.recut_pack([1, S.cuts[0][1] + 2, n]), -1), (lambda: e0.recut_pack([0, S.cuts[0][1] + 2, n - 1]), -1),
             (lambda: e0.recut_pack([0, 0, n]), -1), (lambda: e0.recut_pack([0, n, n]), -1),
             (lambda: e0.recut_apply(3, 3, None, 0), -1), (lambda: e0.recut_apply(0, n + 1, None, 0), -1),
             (lambda: e0.recut_apply(-1, 5, None, 0), -1)]
    # rank 1's departing rows under flat, applied on rank 1 itself: it does not own them
    c1 = e1.recut_pack(flat)
    assert c1[0] > 0
    b1 = _buf(int(c1.sum()) * RB)
    e1.recut_pack(flat, b1)
    cases.append((lambda: e1.recut_apply(flat[1], flat[2], b1, int(c1[0])), -1))
    cases.append((lambda: e0.recut_pack([0, S.cuts[0][1] - 1, n], _buf(RB)), -3))   # more departing rows than the buffer holds
    for call, code in cases:
        with pytest.raises(capi.MpmbError) as ex:
            call()
        assert ex.value.code == code
        for e, snap in zip(S.eng, snaps):
            _assert_unchanged(e, snap)
    e0.sort_particles_and_populate_grid()                                      # inside a substep
    for call in (e0.layer_counts, lambda: e0.recut_pack(flat), lambda: e0.recut_apply(0, flat[1], None, 0)):
        with pytest.raises(capi.MpmbError) as ex:
            call()
        assert ex.value.code == -4
    S.close(); ref.close()


def test_configured_capacity_too_small_changes_nothing():
    scene, st = _scene()
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    n = slab.tile_layers(scene["res"][2])
    cuts = slab.slab_partition(tz, n, 2)
    mine = np.nonzero(tz < cuts[0][1])[0]
    eng = []
    for rank, (z0, z1) in enumerate(cuts):
        sel = np.nonzero((tz >= z0) & (tz < z1))[0]
        e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], rank=rank, world=2, tile_z0=z0, tile_z1=z1,
                        migrate_capacity=4096, capacity=len(mine) + 10 if rank == 0 else 0)
        e.set_material(0, int(scene["mat_kind"][0]), scene["mat_params"][0])
        e.set_planes(scene["planes"], scene["friction"])
        e.set_id_base(0 if rank == 0 else len(mine))
        e.upload(*(st[k][sel] for k in KEYS))
        eng.append(e)
    flat = [0, cuts[0][1] + 2, n]                                             # rank 0 would take rank 1's lowest layers
    c1 = eng[1].recut_pack(flat)
    b1 = _buf(int(c1.sum()) * RB)
    eng[1].recut_pack(flat, b1)
    assert c1[0] > 10
    snap = _snapshot(eng[0])
    with pytest.raises(capi.MpmbError) as ex:
        eng[0].recut_apply(flat[0], flat[1], b1, int(c1[0]))
    assert ex.value.code == -3
    _assert_unchanged(eng[0], snap)
    assert eng[0].tile_range() == cuts[0]
    for e in eng:
        e.close()


# ---- two GPUs: one process per rank, slab.rebalance over NCCL, then whole substeps

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
    x, _, _ = scenes.lattice_block(32, (11, 18, 14), (21, 28, 4 * cuts[0][1] - 1), jitter=0.2, seed=51)
    A = _sand(x, 52)
    first = slab.global_id_end(e, dist)
    slab.append_particles(e, A, first, dist)
    run(6)
    torch.cuda.synchronize()
    old, new, moved = slab.rebalance(e, rank, world, dist)
    same = slab.rebalance(e, rank, world, dist)
    run(10)
    torch.cuda.synchronize()
    e.synchronize()
    got = e.download()
    ids = got["id"].astype(np.int64)
    order = np.concatenate([np.nonzero((tz >= a) & (tz < b))[0] for a, b in cuts])
    got["gid"] = np.where(ids < len(st["x"]), order[np.minimum(ids, len(st["x"]) - 1)], ids)
    np.savez(out_path % rank, **got, first=first, old=np.array(old), new=np.array(new), moved=moved, same_moved=same[2],
             range=np.array(e.tile_range()), id_end=slab.global_id_end(e, dist))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


@pytest.mark.needs_cuda
@pytest.mark.parametrize("transport", ["nccl", "peer"])
def test_two_ranks_rebalance_over_nccl_then_whole_substeps(tmp_path, transport):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out_path = str(tmp_path / "rank%d.npz")
    mp.spawn(_spawn_worker, args=(2, _free_port(), transport, out_path), nprocs=2, join=True)
    scene, st = _scene()
    cuts = slab.slab_partition(slab.base_tile_z(st["x"][:, 2], scene["dx"]), slab.tile_layers(scene["res"][2]), 2)
    x, _, _ = scenes.lattice_block(32, (11, 18, 14), (21, 28, 4 * cuts[0][1] - 1), jitter=0.2, seed=51)
    A = _sand(x, 52)
    ref = T.make_engine(scene, st)
    ref.substep(6)
    assert ref.append(*(A[k] for k in KEYS)) == len(st["x"])
    ref.substep(16)
    want = ref.download()
    ref.close()
    parts = [dict(np.load(out_path % r)) for r in range(2)]
    for r, p in enumerate(parts):
        assert np.array_equal(p["old"], parts[0]["old"]) and np.array_equal(p["new"], parts[0]["new"])
        assert not np.array_equal(p["new"], p["old"]) and int(p["moved"]) > 0 and int(p["same_moved"]) == 0
        assert tuple(p["range"]) == tuple(p["new"][r])
        assert int(p["id_end"]) == len(st["x"]) + len(A["x"])
    _assert_match(parts, want)
