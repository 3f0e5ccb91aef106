"""Rigid-coupled scenes on z-slab ranks: every rank rasterises the colour field of every body, transfers its own tiles and sums
the bodies' impulses over the ranks after each transfer, so the bodies stay bit-identical on every rank; a particle's colour
state travels with it through the migration and the re-cut.  W = 2 and W = 4 slabs in one process on one device, cut through the
paddle and the jelly it stirs, against one engine of the same scene."""
import os

import numpy as np
import pytest

from taichi_mpm_b200 import capi, slab
from taichi_mpm_b200 import mpm as mpm_mod, scenes
from tests.test_gpu_rigid_motion import GRAVITY
from tests.test_gpu_rigid_parity import MAX_FLIPS, TOL_CHAIN_BODY

pytestmark = pytest.mark.gpu
SIMT = os.environ.get("MPMB_SIMT", "") == "1"
NSUB = 40


class _DevBuf:
    """A device byte buffer: a torch CUDA tensor, or host memory under the SIMT emulator (device memory is host memory there)."""

    def __init__(self, n):
        if SIMT:
            self.a = np.zeros(max(int(n), 16), np.uint8)
        else:
            import torch
            self.a = torch.zeros(max(int(n), 16), dtype=torch.uint8, device="cuda")

    def data_ptr(self):
        return self.a.ctypes.data if SIMT else self.a.data_ptr()

    def numel(self):
        return len(self.a) if SIMT else self.a.numel()

    def element_size(self):
        return 1


def _paddle_scene(res=32):
    """The scene of test_gpu_rigid_motion._paddle_scene (a scripted paddle stirring a jelly block, a free box falling onto a
    floor plane with level-set collision), with the paddle centred on the tile boundary z = 0.5, so that a cut there runs
    through the body and the particles it colours."""
    m = mpm_mod.MPM(res=(res, res, res), base_delta_t=1e-4, gravity=GRAVITY, penalty=1e3, rigid_body_levelset_collision=True)
    ls = m.create_levelset()
    ls.add_plane((0, 1, 0), -0.25)
    ls.set_friction(0.4)
    m.set_levelset(ls, False)
    lo, hi = int(0.3 * res), int(0.6 * res)
    m.add_particles(type="jelly", benchmark_block=((lo, int(0.25 * res) + 1, lo), (hi, int(0.45 * res), hi)), density=400.0, jitter=0.2, E=2e4)
    m.add_particles(type="rigid", tris=scenes.plate_mesh(0.02, 0.1, axis=0), codimensional=True, friction=0.3,
                    scripted_position=lambda t: (0.33 + 0.8 * t, 0.36, 0.5), scripted_rotation=lambda t: (0.0, 400.0 * t, 10.0))
    m.add_particles(type="rigid", tris=scenes.box_mesh((0.04, 0.03, 0.04)), codimensional=False, density=400.0, friction=0.3,
                    initial_position=(0.7, 0.285, 0.6), initial_velocity=(-0.3, -1.0, 0.0), initial_rotation=(10.0, 20.0, 5.0),
                    angular_damping=0.5, restitution=0.2)
    m._push()
    return m


def _scene_parts():
    """The paddle scene's particles (by id), bodies, motion rows and NSUB script entries, taken from the mirror.  The jelly on
    either side of the paddle moves along z in opposite directions, so coloured particles cross the cut z = 0.5 both ways."""
    m = _paddle_scene()
    st = m.engine.download()
    st["v"][:, 2] = np.where(st["x"][:, 0] < 0.33, 2.0, -2.0).astype(np.float32)
    rec = m._rigid_records()
    rows = [{}] + [b.motion_record() for b in m.rigids]
    h, t = np.float32(m.base_delta_t), np.float32(m.current_t)
    clocks = []
    for _ in range(NSUB):
        clocks.append(float(t) + float(h))
        t = np.float32(t + h)
    table = np.zeros((NSUB, len(m.rigids) + 1, capi.RIGID_SCRIPT_STRIDE))
    for k, b in enumerate(m.rigids):
        if b.pos_func is not None or b.rot_func is not None:
            table[:, k + 1] = b.script_poses(clocks, float(h))
    return m, st, rec, rows, table


CUTS = {1: [(0, 10)], 2: [(0, 4), (4, 10)], 4: [(0, 3), (3, 4), (4, 5), (5, 10)]}   # tile layers; z = 0.5 is the boundary 3 | 4


def _reference(n):
    """One engine (world == 1) of the same scene, built the same way, n substeps in one call (graph replay)."""
    (e,), cuts, n_p, rec = _slabs(1)
    e.substep(n)
    out = e.download()
    out.update(states=e.get_particle_cdf(n_p)["states"][out["id"].astype(np.int64)], body=e.get_rigid_state(len(rec["inv_mass"])))
    e.close()
    return out


def _slabs(world):
    """world engines of the paddle scene, cut through the paddle and the particles it stirs; ids are the mirror's."""
    m, st, rec, rows, table = _scene_parts()
    dx = m.delta_x
    assert np.array_equal(st["id"], np.arange(len(st["id"])))
    cuts = CUTS[world]
    n = len(st["id"])
    eng = []
    for r, (z0, z1) in enumerate(cuts):
        # a configured capacity: the top rank of W = 4 starts empty and must still run every stage (and take immigrants)
        e = capi.Engine(m.res, dx, m.base_delta_t, m.gravity, True, True, capacity=2 * n, rank=r, world=world, tile_z0=z0, tile_z1=z1,
                        migrate_capacity=4096, halo_capacity=64)
        for g, (kind, prm) in enumerate(m._groups):
            e.set_material(g, kind, prm)
        e.set_planes(m._levelset.planes_grid_units(), m._levelset.friction)
        # every rank gets the whole set and keeps what it owns, particle k with id k (the mirror's): the id end of every rank
        # is then the run's, so an immigrant of any id has a colour entry
        e.append_owned(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"], first_id=0)
        eng.append(e)
    out = []
    for e in eng:
        e.set_rigid(rec)
        e.set_rigid_motion(rows, levelset_collision=True)
        e.set_rigid_script(table)
        out.append(e)
    for r in range(world - 1):   # (no loop on world == 1)
        for k in (0, 1):
            out[r].xchg_connect(k, 1, ptr=out[r + 1].xchg_buffer(k, 0))
            out[r + 1].xchg_connect(k, 0, ptr=out[r].xchg_buffer(k, 1))
    for r in range(world):
        for j in range(world):
            if j != r:
                out[r].rigid_connect(j, ptr=out[j].rigid_mailbox())
    m.engine.close()
    return out, cuts, n, rec


def _reduce(eng, transport, bufs):
    if transport == "mailbox":
        for e in eng:
            e.rigid_send()
        for e in eng:
            e.rigid_recv()
    else:   # host transport: every rank's partials packed, gathered in rank order, summed by every rank
        nbytes = eng[0].rigid_impulse_bytes()
        for r, e in enumerate(eng):
            e.rigid_impulse_pack(bufs.data_ptr() + r * nbytes)
        for e in eng:
            e.rigid_impulse_apply(bufs.data_ptr())


def _substep(eng, transport, bufs):
    world = len(eng)
    faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < world] for r in range(world)]
    for e in eng:
        e.sort_particles_and_populate_grid(); e.rasterize()
    _reduce(eng, transport, bufs)
    for r, e in enumerate(eng):
        for f in faces[r]:
            e.halo_send(f)
    for r, e in enumerate(eng):
        for f in faces[r]:
            e.halo_recv(f)
    for e in eng:
        e.resample()
    _reduce(eng, transport, bufs)
    for r, e in enumerate(eng):
        for f in faces[r]:
            e.migrate_send(f)
    for r, e in enumerate(eng):
        for f in faces[r]:
            e.migrate_recv(f)


def _union(eng, n):
    parts = [e.download() for e in eng]
    for p, e in zip(parts, eng):
        p["states"] = e.get_particle_cdf(n)["states"][p["id"].astype(np.int64)]
    u = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    o = np.argsort(u["id"])
    return {k: v[o] for k, v in u.items()}, parts


def _bodies_identical(eng, nb):
    raw = [e.get_rigid_state(nb) for e in eng]
    for r in raw[1:]:
        for k in raw[0]:
            assert raw[0][k].tobytes() == r[k].tobytes(), k
    return raw[0]


def _check_against_one_engine(u, body, ref, rec):
    assert np.array_equal(u["id"], ref["id"])
    ex = np.abs(u["x"] - ref["x"]).max()
    ev = np.abs(u["v"] - ref["v"]).max() / np.abs(ref["v"]).max()
    flips = np.count_nonzero(u["states"] != ref["states"])
    print("x %.3g  v %.3g (relative)  state flips %d of %d" % (ex, ev, flips, len(u["id"])))
    assert ex <= 2e-6 and ev <= 5e-4          # the slab tolerances of test_gpu_slab.py
    assert flips <= MAX_FLIPS * len(u["id"])
    for k in range(1, len(body["position"])):   # the body bounds of the chained-oracle runs (test_gpu_rigid_parity)
        ep = np.abs(ref["body"]["position"][k] - body["position"][k]).max()
        evb = np.abs(ref["body"]["velocity"][k] - body["velocity"][k]).max() / max(np.abs(ref["body"]["velocity"][k]).max(), 1e-7)
        print("body", k, "position", ep, "velocity", evb)
        assert ep <= 1.2e-7 and evb <= TOL_CHAIN_BODY


@pytest.mark.parametrize("world", [2, 4])
def test_slabs_with_bodies_match_one_engine_and_states_travel(world):
    ref = _reference(NSUB)
    eng, cuts, n, rec = _slabs(world)
    owner = np.full(n, -1)
    for r, e in enumerate(eng):
        owner[e.download()["id"].astype(np.int64)] = r
    crossed = {+1: 0, -1: 0}
    for _ in range(NSUB):
        _substep(eng, "mailbox", None)
        _bodies_identical(eng, len(rec["inv_mass"]))
        states = [e.get_particle_cdf(n)["states"] for e in eng]
        now = np.full(n, -1)
        for r, e in enumerate(eng):
            now[e.download()["id"].astype(np.int64)] = r
        moved = np.nonzero((owner >= 0) & (now >= 0) & (owner != now))[0]
        for i in moved:   # the state word arrived intact: the receiving rank holds what the sending rank packed
            assert states[now[i]][i] == states[owner[i]][i], (i, owner[i], now[i])
            if states[now[i]][i]:
                crossed[int(np.sign(now[i] - owner[i]))] += 1
        owner = now
    print("cuts", cuts, "migrants with a colour state, up / down:", crossed)
    assert crossed[+1] > 0 and crossed[-1] > 0, "no coloured particle crossed a cut in both directions"
    u, _ = _union(eng, n)
    body = _bodies_identical(eng, len(rec["inv_mass"]))
    _check_against_one_engine(u, body, ref, rec)
    for e in eng:
        e.close()


def test_host_transport_agrees_with_the_mailboxes():
    world = 2
    runs = {}
    for transport in ("mailbox", "host"):
        eng, cuts, n, rec = _slabs(world)
        bufs = _DevBuf(world * eng[0].rigid_impulse_bytes())
        for _ in range(NSUB // 2):
            _substep(eng, transport, bufs)
        u, _ = _union(eng, n)
        runs[transport] = (u, _bodies_identical(eng, len(rec["inv_mass"])))
        for e in eng:
            e.close()
    (a, ba), (b, bb) = runs["mailbox"], runs["host"]
    assert np.array_equal(a["id"], b["id"])
    assert np.abs(a["x"] - b["x"]).max() <= 1e-5
    assert np.abs(a["v"] - b["v"]).max() <= 1e-3 * np.abs(b["v"]).max()
    assert np.abs(ba["position"] - bb["position"]).max() <= 1e-6


def _batch(n_side=12):
    """Particles appended between substeps: a layer above the block and a layer sunk into the floor (phi < 0), which the
    level-set deletion then removes."""
    g = 0.32 + 0.26 * np.arange(n_side) / n_side
    X, Z = np.meshgrid(g, g, indexing="ij")
    x = np.concatenate([np.stack([X.ravel(), np.full(X.size, y), Z.ravel()], 1) for y in (0.47, 0.235)]).astype(np.float32)
    m = len(x)
    vol = np.full(m, (1 / 32) ** 3 / 8, np.float32)
    F = np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (m, 1))
    return dict(x=x, v=np.zeros((m, 3), np.float32), mass=vol * 400, vol=vol, F=F, b=np.zeros((m, 9), np.float32),
                ps=np.zeros(m, np.float32), group=np.zeros(m, np.int32))


def _edit(engines, first_id):
    """The same append and level-set deletion on every engine; returns (kept, deleted) over all of them."""
    bt = _batch()
    kept = sum(slab.append_particles(e, bt, first_id) for e in engines)
    deleted = sum(slab.delete_inside_levelset(e) for e in engines)
    return kept, deleted


def test_recut_and_edits_with_bodies_follow_one_engine():
    world, n_before, n_after = 2, 10, 6
    ref_e, _, n, rec = (lambda t: (t[0][0], t[1], t[2], t[3]))(_slabs(1))
    ref_e.substep(n_before)
    eng, cuts, _, _ = _slabs(world)
    for _ in range(n_before):
        _substep(eng, "mailbox", None)
    before, _ = _union(eng, n)
    # re-cut: the cut moves one tile layer up, the particles of that layer go from rank 1 to rank 0 with their records
    z = cuts[0][1] + 1
    new = [(0, z), (z, cuts[1][1])]
    flat = [0, z, cuts[1][1]]
    packed = []
    for e in eng:
        counts = e.recut_pack(flat)
        buf = _DevBuf(int(counts.sum()) * capi.RECORD_BYTES)
        e.recut_pack(flat, buf)
        packed.append((buf, counts))
    assert packed[1][1][0] > 0
    for r, e in enumerate(eng):
        e.recut_apply(*new[r], packed[1 - r][0], int(packed[1 - r][1][r]))
    after, _ = _union(eng, n)
    assert np.array_equal(before["id"], after["id"])
    assert np.array_equal(before["states"], after["states"]) and np.count_nonzero(after["states"]) > 0
    # append + delete with bodies present, the same edit on the slabs and on the one engine
    got, want = _edit(eng, n), _edit([ref_e], n)
    assert got == want and want[0] > 0 and want[1] > 0, (got, want)
    n_all = n + len(_batch()["x"])
    for _ in range(n_after):
        _substep(eng, "mailbox", None)
        body = _bodies_identical(eng, len(rec["inv_mass"]))
    ref_e.substep(n_after)
    ref = ref_e.download()
    ref.update(states=ref_e.get_particle_cdf(n_all)["states"][ref["id"].astype(np.int64)], body=ref_e.get_rigid_state(len(rec["inv_mass"])))
    ref_e.close()
    u, _ = _union(eng, n_all)
    assert np.count_nonzero(u["id"] >= n) > 0              # appended particles live on
    _check_against_one_engine(u, body, ref, rec)
    for e in eng:
        e.close()


def test_error_codes_on_rigid_slab_ranks():
    eng, cuts, n, rec = _slabs(2)
    e0, e1 = eng
    for e in eng:
        e.sort_particles_and_populate_grid(); e.rasterize()
    with pytest.raises(capi.MpmbError) as ex:
        e0.resample()                                   # before the P2G impulse reduction
    assert ex.value.code == -4
    with pytest.raises(capi.MpmbError) as ex:
        e0.rigid_recv()                                  # a receive without this rank's send
    assert ex.value.code == -4
    _reduce(eng, "mailbox", None)
    for e in eng:
        e.resample()
    with pytest.raises(capi.MpmbError) as ex:
        e0.sort_particles_and_populate_grid()            # before the G2P impulse reduction
    assert ex.value.code == -4
    _reduce(eng, "mailbox", None)
    for e in eng:
        e.close()
    # mpmb_substep with the halo peers but not the mailboxes connected: refused, nothing enqueued
    m, st, rec, rows, table = _scene_parts()
    nb = len(rec["inv_mass"])
    tz = slab.base_tile_z(st["x"][:, 2], m.delta_x)
    cuts = slab.slab_partition(tz, slab.tile_layers(m.res[2]), 2)
    es = []
    for r, (z0, z1) in enumerate(cuts):
        e = capi.Engine(m.res, m.delta_x, m.base_delta_t, m.gravity, True, True, rank=r, world=2, tile_z0=z0, tile_z1=z1,
                        migrate_capacity=4096, halo_capacity=64)
        mine = np.nonzero((tz >= z0) & (tz < z1))[0]
        e.upload(*(st[k][mine] for k in ("x", "v", "mass", "vol", "F", "b", "ps", "group")))
        e.set_rigid(rec)
        es.append(e)
    for k in (0, 1):
        es[0].xchg_connect(k, 1, ptr=es[1].xchg_buffer(k, 0))
        es[1].xchg_connect(k, 0, ptr=es[0].xchg_buffer(k, 1))
    launches = es[0].get_counters()["kernel_launches"]
    with pytest.raises(capi.MpmbError) as ex:
        es[0].substep(1)
    assert ex.value.code == -4
    assert es[0].get_counters()["kernel_launches"] == launches
    with pytest.raises(capi.MpmbError) as ex:
        es[0].async_init((4, 4, 4), 32.0)                # AsyncMPM stays refused on slab ranks
    assert ex.value.code == -4
    m.engine.close()
    for e in es:
        e.close()


# ------------------------------------------------------------------------------------------- bodies that take impulses
# The scenes of test_gpu_rigid_parity's chained-oracle runs (a plate through a strained jelly block), cut into z slabs through
# the block and the plate, against the same chained fp64 oracle and its bounds.  The free plate takes the particles' impulses
# summed over the ranks: a missing, partial or misplaced partial sum moves its trajectory off the oracle's.
def _golden_slabs(scene, st, rigid, world):
    n = len(st["x"])
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    cuts = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)
    eng = []
    for r, (z0, z1) in enumerate(cuts):
        e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], scene.get("particle_gravity", 1), scene.get("clean_boundary", True),
                        capacity=2 * n, rank=r, world=world, tile_z0=z0, tile_z1=z1, migrate_capacity=4096, halo_capacity=64)
        for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
            e.set_material(g, int(k), p)
        if scene.get("planes") is not None:
            e.set_planes(scene["planes"], scene["friction"])
        e.append_owned(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"], first_id=0)
        e.set_rigid(rigid)
        eng.append(e)
    for r in range(world - 1):
        for k in (0, 1):
            eng[r].xchg_connect(k, 1, ptr=eng[r + 1].xchg_buffer(k, 0))
            eng[r + 1].xchg_connect(k, 0, ptr=eng[r].xchg_buffer(k, 1))
    for r in range(world):
        for j in range(world):
            if j != r:
                eng[r].rigid_connect(j, ptr=eng[j].rigid_mailbox())
    occupied = [int(((tz >= a) & (tz < b)).sum()) for a, b in cuts]
    assert sum(1 for c in occupied if c) >= 2, cuts
    return eng


class _Parts:
    """The overlap schedule with host-moved bytes: boundary-layer P2G, halo pack, interior P2G, the P2G impulse reduction
    (host transport), interior G2P, halo unpack, boundary G2P, the G2P reduction, migration."""

    def __init__(self, eng):
        self.eng = eng
        self.imp = _DevBuf(len(eng) * eng[0].rigid_impulse_bytes())
        self.halo = [[_DevBuf(e.halo_bytes()) for _ in (0, 1)] for e in eng]
        self.mig = [[_DevBuf(e.migrate_bytes()) for _ in (0, 1)] for e in eng]

    def __call__(self):
        eng, W = self.eng, len(self.eng)
        faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < W] for r in range(W)]
        nbr = lambda r, f: r - 1 if f == 0 else r + 1
        for e in eng:
            e.sort_particles_and_populate_grid(); e.rasterize_part(1)
        for r, e in enumerate(eng):
            for f in faces[r]:
                e.halo_pack(f, self.halo[r][f].data_ptr())
        for e in eng:
            e.rasterize_part(2)
        _reduce(eng, "host", self.imp)
        for e in eng:
            e.resample_part(2)
        for r, e in enumerate(eng):
            for f in faces[r]:
                e.halo_unpack(f, self.halo[nbr(r, f)][1 - f].data_ptr())
        for e in eng:
            e.resample_part(1)
        _reduce(eng, "host", self.imp)
        for r, e in enumerate(eng):
            for f in faces[r]:
                e.migrate_pack(f, self.mig[r][f].data_ptr())
        for r, e in enumerate(eng):
            for f in faces[r]:
                e.migrate_unpack(f, self.mig[nbr(r, f)][1 - f].data_ptr())


def _stepper(eng, schedule):
    return _Parts(eng) if schedule == "parts" else (lambda: _substep(eng, "mailbox", None))


def _states_by_id(eng, u, n):
    out = np.zeros(n, np.uint32)
    out[u["id"].astype(np.int64)] = u["states"]
    return out


@pytest.mark.parametrize("world,schedule", [(2, "whole"), (4, "whole"), (2, "parts"), (4, "parts")])
def test_free_plate_on_slabs_against_the_chained_oracle(world, schedule):
    from oracle import pyoracle as O
    from tests.test_gpu_rigid_motion import _host_advect, _host_bodies, _motion
    from tests.test_gpu_rigid_parity import TOL_CHAIN_BODY, _chain_errors, _kind_scene, _rel
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    n, nsub = len(st["x"]), 10
    dt = float(np.float32(scene["dt"]))
    eng = _golden_slabs(scene, st, rigid, world)
    for e in eng:
        e.set_rigid_motion(_motion(_host_bodies(rigid)))
    step = _stepper(eng, schedule)
    b = _host_bodies(rigid)[0]
    cur, r, t = dict(st, states=np.zeros(n, np.uint32)), rigid, 0.0
    worst = dict(position=0.0, velocity=0.0, angular_velocity=0.0)
    nb = len(rigid["inv_mass"])
    for k in range(nsub):
        step()
        rs = _bodies_identical(eng, nb)
        cur, _, _, rv, _ = O.substep_coupled(scene, cur, r, np.float64)
        b.velocity, b.angular_velocity = rv["velocity"][1].copy(), rv["angular_velocity"][1].copy()
        _host_advect(b, t, dt)
        t += dt
        r = dict(rigid, position=rigid["position"].copy(), rot=rigid["rot"].copy(), velocity=rigid["velocity"].copy(),
                 angular_velocity=rigid["angular_velocity"].copy(), inv_inertia=rigid["inv_inertia"].copy())
        r["position"][1], r["velocity"][1], r["angular_velocity"][1] = b.position, b.velocity, b.angular_velocity
        r["rot"][1] = b.rotation.T.reshape(9)
        r["inv_inertia"][1] = (b.rotation @ b.inv_inertia_body @ b.rotation.T).T.reshape(9)
        for key in worst:
            worst[key] = max(worst[key], _rel(rs[key][1], getattr(b, key)) if key != "position" else float(np.abs(rs[key][1] - b.position).max()))
    u, _ = _union(eng, n)
    for e in eng:
        e.close()
    print("free plate on %d slabs (%s), body trajectory" % (world, schedule), worst)
    _chain_errors(u, dict(states=_states_by_id(eng, u, n)), cur, "free plate, %d slabs, %s" % (world, schedule))
    assert np.abs(b.velocity - rigid["velocity"][1]).max() > 1e-2
    assert worst["position"] <= 1.2e-7 and worst["velocity"] <= TOL_CHAIN_BODY and worst["angular_velocity"] <= TOL_CHAIN_BODY, worst


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("mode", ["host", "device"])
def test_scripted_plate_on_slabs_against_the_chained_oracle(mode, world):
    # host: the per-substep contract on every rank (set_rigid_state with the pose of the substep); device: device motion with
    # the script table, the advance after the G2P reduction
    from oracle import pyoracle as O
    from tests.test_gpu_rigid_motion import _host_bodies, _motion, _scripted_pose_table
    from tests.test_gpu_rigid_parity import _chain_errors, _kind_scene
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "kinematic")
    rigid["velocity"] = rigid["velocity"].copy()
    rigid["velocity"][1] = (2.0, -0.5, 1.0)
    n, nsub = len(st["x"]), 20
    dt = float(np.float32(scene["dt"]))
    bodies = _host_bodies(rigid)
    table, _ = _scripted_pose_table(bodies, nsub, dt)

    def pose(k):
        r = dict(rigid)
        if k:
            for key, sl in (("position", slice(0, 3)), ("rot", slice(3, 12)), ("velocity", slice(12, 15)), ("angular_velocity", slice(15, 18))):
                r[key] = rigid[key].copy()
                r[key][1:] = table[k - 1, 1:, sl].astype(np.float32)
        return r
    eng = _golden_slabs(scene, st, rigid, world)
    if mode == "device":
        for e in eng:
            e.set_rigid_motion(_motion(bodies))
            e.set_rigid_script(table)
    for k in range(nsub):
        if mode == "host":
            for e in eng:
                e.set_rigid_state(pose(k))
        _substep(eng, "mailbox", None)
        _bodies_identical(eng, len(rigid["inv_mass"]))
    u, _ = _union(eng, n)
    for e in eng:
        e.close()
    cur = dict(st, states=np.zeros(n, np.uint32))
    for k in range(nsub):
        cur, _, _, _, _ = O.substep_coupled(scene, cur, pose(k), np.float64)
    assert (cur["states"] != 0).sum() > 500
    _chain_errors(u, dict(states=_states_by_id(eng, u, n)), cur, "scripted plate, %d slabs, %s" % (world, mode))


# ------------------------------------------------------------------------------------------- two processes, two GPUs
def _spawn_worker(rank, world, port, transport, out_path):
    import torch
    import torch.distributed as dist
    from tests.test_gpu_rigid_motion import _host_bodies, _motion
    from tests.test_gpu_rigid_parity import _kind_scene
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    tz = slab.base_tile_z(st["x"][:, 2], scene["dx"])
    z0, z1 = slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)[rank]
    mine = np.nonzero((tz >= z0) & (tz < z1))[0]
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], 1, True, device=rank, capacity=2 * len(tz), rank=rank, world=world,
                    tile_z0=z0, tile_z1=z1, migrate_capacity=4096, halo_capacity=64)
    e.set_stream(torch.cuda.current_stream().cuda_stream)
    for g, (k, p) in enumerate(zip(scene["mat_kind"], scene["mat_params"])):
        e.set_material(g, int(k), p)
    # per-rank upload: rank r's particles get ids id_base .. (the run's id end is shared by connect_peers / SlabRunner)
    counts = [int(((tz >= a) & (tz < b)).sum()) for a, b in slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)]
    e.set_id_base(sum(counts[:rank]))
    e.upload(*(st[k][mine] for k in ("x", "v", "mass", "vol", "F", "b", "ps", "group")))
    e.set_rigid(rigid)
    e.set_rigid_motion(_motion(_host_bodies(rigid)))
    if transport == "ipc":
        slab.connect_peers(e, rank, world, dist)
        e.substep(10)                # whole substeps, mailbox reductions inside the replayed graphs
    else:
        slab.SlabRunner(slab.EngineAdapter(e), rank, world, torch.device("cuda", rank), dist=dist).substep(10)
    torch.cuda.synchronize()
    got = e.download()
    order = np.concatenate([np.nonzero((tz >= a) & (tz < b))[0] for a, b in slab.slab_partition(tz, slab.tile_layers(scene["res"][2]), world)])
    got["gid"] = order[got["id"].astype(np.int64)]
    body = e.get_rigid_state(len(rigid["inv_mass"]))
    np.savez(out_path % rank, **got, **{"body_" + k: v for k, v in body.items()})
    dist.barrier()
    e.close()
    dist.destroy_process_group()


@pytest.mark.needs_cuda
@pytest.mark.parametrize("transport", ["ipc", "nccl"])
def test_two_processes_with_a_free_plate_match_one_engine(tmp_path, transport):
    if SIMT:
        pytest.skip("needs real devices")
    import socket
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from tests import common as T
    from tests.test_gpu_rigid_motion import _host_bodies, _motion
    from tests.test_gpu_rigid_parity import _kind_scene
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out_path = str(tmp_path / "rank%d.npz")
    mp.spawn(_spawn_worker, args=(2, port, transport, out_path), nprocs=2, join=True)
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    e = T.make_engine(scene, st)
    e.set_rigid(rigid)
    e.set_rigid_motion(_motion(_host_bodies(rigid)))
    e.substep(10)
    ref, body = e.download(), e.get_rigid_state(len(rigid["inv_mass"]))
    e.close()
    parts = [np.load(out_path % r) for r in range(2)]
    for k in body:
        assert parts[0]["body_" + k].tobytes() == parts[1]["body_" + k].tobytes(), k
    gid = np.concatenate([p["gid"] for p in parts])
    o = np.argsort(gid)
    assert np.array_equal(gid[o], ref["id"].astype(np.int64))
    assert np.abs(np.concatenate([p["x"] for p in parts])[o] - ref["x"]).max() <= 2e-6
    assert np.abs(parts[0]["body_position"][1] - body["position"][1]).max() <= 1.2e-7
