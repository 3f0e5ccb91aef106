"""Rigid bodies advanced on the device (mpmb_set_rigid_motion / mpmb_set_rigid_script): advect_rigid_bodies and
rigid_body_levelset_collision against HostRigidBody (the fp64 host reference), whole frames against the per-substep host loop,
CUDA-graph replay with bodies, the script table and the error codes.  Runs on the SIMT emulator too
(tests/test_rigid_motion_simt.py; the emulator has no graphs)."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from taichi_mpm_b200 import capi, mpm as mpm_mod, rigid as rigid_mod, scenes
from tests import common as T

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_rigid_golden", os.path.join(HERE, "golden", "make_rigid_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

GRAVITY = (0.0, -10.0, 0.0)


def _f32(a):
    return np.asarray(np.asarray(a, np.float32), np.float64)


def _host_bodies(rigid, t0=0.0):
    """HostRigidBody objects for the bodies of a make_rigid dict, every input rounded to what the engine receives (fp32).
    Bodies with zero inverse mass are scripted (a straight line at their velocity, the rotation held); free bodies get damping,
    a rotation axis (body 1) and restitution."""
    out = []
    for b in range(1, len(rigid["inv_mass"])):
        hb = rigid_mod.HostRigidBody.__new__(rigid_mod.HostRigidBody)
        hb.position, hb.velocity, hb.angular_velocity = _f32(rigid["position"][b]), _f32(rigid["velocity"][b]), _f32(rigid["angular_velocity"][b])
        hb.rotation = _f32(rigid["rot"][b]).reshape(3, 3).T
        hb.frictions = tuple(float(f) for f in rigid["frictions"][b])
        hb.restitution = float(np.float32(0.3))
        hb.rot_func = None
        if rigid["inv_mass"][b] == 0:
            p0, v0 = hb.position.copy(), hb.velocity.copy()
            hb.pos_func = lambda t, p0=p0, v0=v0: p0 + v0 * (t - t0)
            hb.mass, hb.inv_mass, hb.inv_inertia_body = 1.0, 0.0, np.zeros((3, 3))
            hb.rotation_axis, hb.linear_damping, hb.angular_damping = np.zeros(3), 0.0, 0.0
        else:
            hb.pos_func = None
            hb.mass = float(np.float32(1.0 / float(rigid["inv_mass"][b])))
            hb.inv_mass = 1.0 / hb.mass
            Iw = _f32(rigid["inv_inertia"][b]).reshape(3, 3).T
            hb.inv_inertia_body = _f32(hb.rotation.T @ Iw @ hb.rotation)
            hb.rotation_axis = _f32((0.2, 1.0, 0.1)) if b == 1 else np.zeros(3)
            hb.linear_damping, hb.angular_damping = float(np.float32(0.5)), float(np.float32(0.8))
        out.append(hb)
    return out


def _scripted_pose_table(bodies, n, dt, t0=0.0):
    """The script table the host hands over (mpmb_set_rigid_script) for n substeps from t0: scripted bodies follow pos_func."""
    table = np.zeros((n, len(bodies) + 1, capi.RIGID_SCRIPT_STRIDE))
    clocks, t = [], np.float32(t0)
    for _ in range(n):
        clocks.append(float(t) + float(dt))
        t = np.float32(t + np.float32(dt))
    for k, b in enumerate(bodies):
        if b.pos_func is not None:
            table[:, k + 1] = b.script_poses(clocks, float(dt))
            table[:, k + 1, 3:12] = b.rotation.T.reshape(9)         # rotation held: scripted, angular velocity 0
    return table, clocks


def _motion(bodies):
    rows = [{}]
    for b in bodies:
        r = b.motion_record()
        if b.pos_func is not None:
            r["scripted_rotation"] = True
        rows.append(r)
    return rows


def _host_advect(b, t, dt):
    """HostRigidBody.advect; a scripted body here holds its rotation (angular velocity 0), as its table entries say."""
    rot = b.rotation.copy()
    b.advect(t, dt, GRAVITY)
    if b.pos_func is not None:
        b.rotation, b.angular_velocity = rot, np.zeros(3)


def _state(e, nb):
    rs = e.get_rigid_state(nb)
    return {k: np.asarray(v, np.float64) for k, v in rs.items()}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _golden(variant):
    scene, st, rigid = G.golden_scene(variant)
    scene = dict(scene, gravity=GRAVITY)
    return scene, st, rigid


@pytest.mark.parametrize("variant", ["kinematic", "dynamic", "two_bodies"])
def test_one_device_substep_matches_host_advect_on_the_read_back_velocities(variant):
    scene, st, rigid = _golden(variant)
    nb = len(rigid["inv_mass"])
    dt = float(np.float32(scene["dt"]))
    legacy = T.make_engine(scene, st)
    legacy.set_rigid(rigid)
    legacy.substep(1)
    rl = _state(legacy, nb)
    legacy.close()
    bodies = _host_bodies(rigid)
    table, _ = _scripted_pose_table(bodies, 1, dt)
    dev = T.make_engine(scene, st)
    dev.set_rigid(rigid)
    dev.set_rigid_motion(_motion(bodies))
    dev.set_rigid_script(table)
    dev.substep(1)
    rd = _state(dev, nb)
    dev.close()
    for k, b in enumerate(bodies):
        b.velocity, b.angular_velocity = rl["velocity"][k + 1], rl["angular_velocity"][k + 1]
        _host_advect(b, 0.0, dt)
        errs = dict(position=_rel(rd["position"][k + 1], b.position), rotation=_rel(rd["rotation"][k + 1], b.rotation),
                    velocity=_rel(rd["velocity"][k + 1], b.velocity), angular_velocity=_rel(rd["angular_velocity"][k + 1], b.angular_velocity))
        print(variant, "body", k + 1, errs)
        for name, err in errs.items():
            assert err <= 1e-6, (name, err)
        if b.pos_func is None:
            assert np.abs(b.velocity - rigid["velocity"][k + 1]).max() > 1e-3       # the transfers and gravity did change it


def _paddle_scene(res=32, levelset_collision=True, no_graph=False, sunk=False):
    """A scripted paddle stirring a jelly block, a free box falling onto a floor plane (the scene of the rigid benchmark, small);
    `sunk`: also a layer of particles inside the floor (y = 0.235, where the level set is negative)."""
    m = mpm_mod.MPM(res=(res, res, res), base_delta_t=1e-4, gravity=GRAVITY, penalty=1e3, rigid_body_levelset_collision=levelset_collision)
    if no_graph:
        m.engine.close()
        m.engine = capi.Engine(m.res, m.delta_x, m.base_delta_t, m.gravity, True, True, no_graph=True)
    ls = m.create_levelset()
    ls.add_plane((0, 1, 0), -0.25)
    ls.set_friction(0.4)
    m.set_levelset(ls, False)
    lo, hi = int(0.3 * res), int(0.6 * res)
    m.add_particles(type="jelly", benchmark_block=((lo, int(0.25 * res) + 1, lo), (hi, int(0.45 * res), hi)), density=400.0, jitter=0.2, E=2e4)
    if sunk:
        m.add_particles(type="jelly", positions=_layer(0.235), density=400.0, E=2e4)
    m.add_particles(type="rigid", tris=scenes.plate_mesh(0.02, 0.1, axis=0), codimensional=True, friction=0.3,
                    scripted_position=lambda t: (0.33 + 0.8 * t, 0.36, 0.45), scripted_rotation=lambda t: (0.0, 400.0 * t, 10.0))
    m.add_particles(type="rigid", tris=scenes.box_mesh((0.04, 0.03, 0.04)), codimensional=False, density=400.0, friction=0.3,
                    initial_position=(0.7, 0.285, 0.6), initial_velocity=(-0.3, -1.0, 0.0), initial_rotation=(10.0, 20.0, 5.0),
                    angular_damping=0.5, restitution=0.2)
    m._push()
    return m


def _layer(y, n_side=24):
    """Particles on a square lattice at height y over x, z in [0.3, 0.6)."""
    g = 0.3 + 0.3 * np.arange(n_side) / n_side
    X, Z = np.meshgrid(g, g, indexing="ij")
    return np.stack([X.ravel(), np.full(X.size, y), Z.ravel()], 1).astype(np.float32)


def _reference_loop(m, n):
    """The mirror's former per-substep path: upload the state, one engine substep, read the velocities back, the level-set
    collision and HostRigidBody.advect on the host."""
    h = np.float32(m.base_delta_t)
    t = np.float32(m.current_t)
    traj = []
    for _ in range(n):
        rec = m._rigid_records()
        if m._rigid_dirty:
            m.engine.set_rigid(rec)
            m._rigid_dirty = False
        else:
            m.engine.set_rigid_state(rec)
        m.engine.substep(1)
        rs = m.engine.get_rigid_state(len(m.rigids) + 1)
        for k, b in enumerate(m.rigids):
            b.velocity = rs["velocity"][k + 1].astype(np.float64)
            b.angular_velocity = rs["angular_velocity"][k + 1].astype(np.float64)
        if m.rigid_body_levelset_collision and getattr(m, "_levelset", None) is not None:
            _levelset_collision(m, rec)
        for b in m.rigids:
            b.advect(float(t), float(h), m.gravity)
        t = np.float32(t + h)
        traj.append([b.position.copy() for b in m.rigids])
    m.current_t = t
    return traj


def _levelset_collision(m, rec):
    ls = m._levelset
    for k, b in enumerate(m.rigids):
        sel = rec["sample_rigid"] == k + 1
        if not sel.any():
            continue
        world = b.position + rec["sample_offset"][sel].astype(np.float64) @ b.rotation.T
        X = world / m.delta_x
        phi = ls.sample(X)
        eps = 0.25
        grad = np.stack([(ls.sample(X + e) - ls.sample(X - e)) / (2 * eps) for e in np.eye(3) * eps], 1)
        nrm = np.linalg.norm(grad, axis=1, keepdims=True)
        b.levelset_collision(world, phi, grad / np.maximum(nrm, 1e-12))


def test_forty_substeps_in_one_call_follow_the_per_substep_host_loop():
    # tolerances: both runs use the same transfers, whose float atomics sum in a different order from run to run.  Measured on an
    # H100 80GB HBM3: body positions 3.6e-5 of the displacement, velocities 5e-8 relative, particle positions 3e-8 (world
    # units), particle velocities 4e-8 relative; the bounds below leave room for that noise growing over 40 coupled substeps
    n = 40
    dev, ref = _paddle_scene(), _paddle_scene()
    y_box0 = ref.rigids[1].position[1]
    traj = _reference_loop(ref, n)
    t_dev = dev._rigid_substeps(n)
    assert t_dev == ref.current_t
    for k in range(2):
        bd, br = dev.rigids[k], ref.rigids[k]
        moved = np.abs(traj[-1][k] - traj[0][k]).max()
        errs = dict(position=np.abs(bd.position - br.position).max() / moved, velocity=_rel(bd.velocity, br.velocity),
                    rotation=np.abs(bd.rotation - br.rotation).max(), angular_velocity=np.abs(bd.angular_velocity - br.angular_velocity).max())
        print("body", k + 1, "moved", moved, errs)
        assert errs["position"] <= 1e-4 and errs["velocity"] <= 1e-3 and errs["rotation"] <= 1e-5
        assert errs["angular_velocity"] <= 1e-3 * max(np.abs(br.angular_velocity).max(), 1.0)
    assert ref.rigids[1].position[1] < y_box0 - 1e-3            # the box fell
    pd, pr = dev.get_particles(), ref.get_particles()
    assert np.array_equal(pd["id"], pr["id"])
    ex, ev = np.abs(pd["x"] - pr["x"]).max(), np.abs(pd["v"] - pr["v"]).max() / np.abs(pr["v"]).max()
    print("particles: x %.3g, v %.3g (relative)" % (ex, ev))
    assert ex <= 1e-5 and ev <= 1e-3


def test_graph_replay_keeps_the_particle_colours_current():
    # graphs on and off: same bodies, same colours, same particles.  (The last substep of a frame always runs from the host,
    # so the colours read back here are that substep's: this compares the replayed substeps through their effect on the state.)
    a, b = _paddle_scene(), _paddle_scene(no_graph=True)
    for m in (a, b):
        m._rigid_substeps(11)
    n = a._n_uploaded
    ca, cb = a.engine.get_particle_cdf(n), b.engine.get_particle_cdf(n)
    assert ca["near"].sum() > 0 and cb["near"].sum() > 0
    assert (ca["states"] != cb["states"]).mean() <= 0.002
    assert (ca["states"] != 0).sum() > 20
    for k in range(2):
        assert np.abs(a.rigids[k].position - b.rigids[k].position).max() <= 1e-5
    pa, pb = a.get_particles(), b.get_particles()
    assert np.abs(pa["x"] - pb["x"]).max() <= 1e-5


def _box_engine(dt=1e-4, restitution=0.0, floor=0.25, y=0.32, particles=True, tilted=True, collide=True):
    """A free box above a floor plane (tilted and spinning, or level and falling straight; floor=None: no level set); a small
    jelly block far from it (or no particles)."""
    res, dx = 32, 1.0 / 32
    e = capi.Engine((res, res, res), dx, dt, GRAVITY, True, True)
    e.set_material(0, scenes.MAT_JELLY, scenes.material_params(scenes.MAT_JELLY))
    if floor is not None:
        e.set_planes(np.array([[0.0, 1.0, 0.0, -floor / dx]], np.float32), 0.4)
    if particles:
        x, mass, vol = scenes.lattice_block(res, (9, 9, 20), (12, 12, 23), 400.0, 0.0, dx=dx)
        st = scenes.make_state(x, mass, vol, scenes.MAT_JELLY, 0, (0.0, 0.0, 0.0))
        e.upload(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
    body = rigid_mod.HostRigidBody(scenes.box_mesh((0.04, 0.03, 0.05)), density=400.0, position=(0.5, y, 0.4),
                                   euler_deg=(8.0, 3.0, 12.0) if tilted else (0, 0, 0), velocity=(0.2, -0.5, 0.0) if tilted else (0.0, -0.5, 0.0),
                                   angular_velocity=(0.5, 0.0, 1.0) if tilted else (0, 0, 0), frictions=(0.3, 0.3), restitution=restitution)
    body.position, body.velocity, body.angular_velocity, body.rotation = (_f32(getattr(body, k)) for k in ("position", "velocity", "angular_velocity", "rotation"))
    body.mass = float(np.float32(body.mass))
    body.inv_mass = 1.0 / body.mass
    body.inv_inertia_body = _f32(body.inv_inertia_body)
    rec = rigid_mod.engine_records([body], dx, 0.0, 20000.0)
    e.set_rigid(rec)
    e.set_rigid_motion([{}, body.motion_record()], levelset_collision=collide)
    return e, body, rec


def test_levelset_impulses_match_host_rigid_body_per_substep():
    # the box starts inside the floor: every substep applies impulses at the samples below it; no particle comes near the box,
    # so only gravity, the impulses and the advance change it
    e, body, rec = _box_engine(y=0.27, particles=True)
    dx, dt = 1.0 / 32, float(np.float32(1e-4))
    ls = mpm_mod.LevelSet((32, 32, 32), dx)
    ls.add_plane((0, 1, 0), -0.25)
    hits = 0
    for s in range(3):
        e.substep(1)
        world = body.position + rec["sample_offset"].astype(np.float64) @ body.rotation.T
        X = world / dx
        phi = ls.sample(X)
        grad = np.stack([(ls.sample(X + d) - ls.sample(X - d)) / 0.5 for d in np.eye(3) * 0.25], 1)
        hits += body.levelset_collision(world, phi, grad / np.maximum(np.linalg.norm(grad, axis=1, keepdims=True), 1e-12))
        body.advect(0.0, dt, GRAVITY)
        rd = _state(e, 2)
        errs = [_rel(rd["velocity"][1], body.velocity), _rel(rd["angular_velocity"][1], body.angular_velocity),
                _rel(rd["position"][1], body.position), _rel(rd["rotation"][1], body.rotation)]
        print("substep", s, errs)
        assert max(errs) <= 1e-5, errs
        # continue from the device's fp32 read-back so that the comparison stays per substep
        body.velocity, body.angular_velocity = rd["velocity"][1], rd["angular_velocity"][1]
        body.position, body.rotation = rd["position"][1], rd["rotation"][1]
        e.set_rigid_state(rigid_mod.state_records([body]))
    assert hits > 10
    e.close()


def test_box_dropped_on_the_floor_comes_to_rest_above_it():
    e, body, rec = _box_engine(dt=1e-3, particles=False)
    e.substep(600)
    rd = _state(e, 2)
    world = rd["position"][1] + rec["sample_offset"].astype(np.float64) @ rd["rotation"][1].T
    print("rest: lowest sample", world[:, 1].min(), "velocity", rd["velocity"][1], "angular", rd["angular_velocity"][1])
    assert world[:, 1].min() > 0.25 - 0.25 / 32 and world[:, 1].min() < 0.25 + 0.25 / 32
    assert np.abs(rd["velocity"][1]).max() < 0.05 and np.abs(rd["angular_velocity"][1]).max() < 0.5
    e.close()


def test_box_with_restitution_bounces():
    ys = {}
    for r in (0.0, 0.5):
        e, body, _ = _box_engine(dt=1e-3, restitution=r, particles=False, y=0.35, tilted=False)
        vy = []
        for _ in range(150):
            e.substep(1)
            vy.append(float(_state(e, 2)["velocity"][1][1]))
        ys[r] = max(vy[60:])
        e.close()
    print("largest upward velocity after the impact:", ys)
    # (with e = 0 the box still rises somewhat: the impulses are applied sample after sample, and the first ones tip it — as the
    # reference's loop does; 0.21 against 0.46 with e = 0.5 on the emulator)
    assert ys[0.5] > 0.3 and ys[0.5] > ys[0.0] + 0.15


def _script_engine(scene, st, rigid):
    bodies = _host_bodies(rigid)
    e = T.make_engine(scene, st)
    e.set_rigid(rigid)
    e.set_rigid_motion(_motion(bodies))
    return e, bodies


def test_script_pose_short_table_and_frames():
    scene, st, rigid = _golden("two_bodies")
    rigid = dict(rigid, inv_mass=rigid["inv_mass"].copy())
    rigid["inv_mass"][1] = 0.0                                   # the plate scripted, the box free
    dt = float(np.float32(scene["dt"]))
    n = 5
    # after n substeps the scripted body sits at the last entry (fp32 of it)
    e, bodies = _script_engine(scene, st, rigid)
    table, _ = _scripted_pose_table(bodies, 2 * n, dt)
    e.set_rigid_script(table)
    e.substep(n)
    rd = e.get_rigid_state(3)
    assert np.array_equal(rd["position"][1], table[n - 1, 1, 0:3].astype(np.float32))
    assert np.array_equal(rd["rotation"][1], table[n - 1, 1, 3:12].reshape(3, 3).T.astype(np.float32))
    assert np.array_equal(rd["velocity"][1], table[n - 1, 1, 12:15].astype(np.float32))
    e.substep(n)                                                  # frame 2: the rest of the table
    two = (e.download(), e.get_rigid_state(3))
    # a table too short for nsub: MPMB_ERR_STATE, nothing enqueued
    p0 = e.download()
    with pytest.raises(capi.MpmbError) as ex:
        e.substep(1)
    assert ex.value.code == -4
    e.set_rigid_script(table[:2])
    with pytest.raises(capi.MpmbError) as ex:
        e.substep(3)
    assert ex.value.code == -4
    p1, r1 = e.download(), e.get_rigid_state(3)
    for k in ("x", "v", "F"):
        assert np.array_equal(p0[k], p1[k]), k
    for k in ("position", "velocity", "rotation"):
        assert np.array_equal(two[1][k], r1[k]), k
    e.close()
    # two frames of n against one frame of 2n
    f, _ = _script_engine(scene, st, rigid)
    f.set_rigid_script(table)
    f.substep(2 * n)
    one = (f.download(), f.get_rigid_state(3))
    f.close()
    assert np.array_equal(one[1]["position"][1], two[1]["position"][1])
    assert _rel(one[1]["position"][2], two[1]["position"][2]) <= 1e-6 and _rel(one[1]["velocity"][2], two[1]["velocity"][2]) <= 1e-4
    assert np.abs(one[0]["x"] - two[0]["x"]).max() <= 2e-6


def test_switching_motion_off_restores_the_pose_held_contract():
    scene, st, rigid = _golden("dynamic")
    e, bodies = _script_engine(scene, st, rigid)
    e.set_rigid_script(np.zeros((4, 2, 18)))
    e.substep(4)
    assert np.abs(e.get_rigid_state(2)["position"][1] - rigid["position"][1]).max() > 1e-5   # advanced
    e.set_rigid_motion([])
    e.set_rigid_state(rigid)
    e.substep(3)
    rs = e.get_rigid_state(2)
    assert np.array_equal(rs["position"][1], rigid["position"][1])            # held over the n substeps
    assert np.array_equal(rs["rotation"][1], rigid["rot"][1].reshape(3, 3).T)
    e.substep(1)                                                            # no script needed any more
    e.close()


def test_error_codes():
    scene, st, rigid = _golden("dynamic")
    e = T.make_engine(scene, st)
    rows = [{}, dict(mass=3.0, inv_inertia_body=np.eye(3))]
    with pytest.raises(capi.MpmbError) as ex:
        e.set_rigid_motion(rows)                                           # before the samples
    assert ex.value.code == -4
    with pytest.raises(capi.MpmbError) as ex:
        e.set_rigid_script(np.zeros((1, 2, 18)))                           # before the motion
    assert ex.value.code == -4
    e.set_rigid(rigid)
    for bad in ([{}], rows + [{}], [{}, dict(mass=float("nan"))], [{}, dict(mass=3.0, inv_inertia_body=np.full((3, 3), np.inf))],
                [{}, dict(mass=0.0)], [{}, dict(mass=3.0, restitution=float("inf"))]):
        with pytest.raises(capi.MpmbError) as ex:
            e.set_rigid_motion(bad)
        assert ex.value.code == -1, bad
    e.set_rigid_motion([{}, dict(mass=3.0, scripted_position=True)])
    assert e.L.mpmb_set_rigid_script(e.h, C.c_int32(-1), None) == -1      # negative length
    assert e.L.mpmb_set_rigid_script(e.h, C.c_int32(2), None) == -1       # NULL table
    bad = np.zeros((2, 2, 18))
    bad[1, 1, 0] = np.nan
    with pytest.raises(capi.MpmbError) as ex:
        e.set_rigid_script(bad)                                            # non-finite scripted part
    assert ex.value.code == -1
    bad[1, 1, 0] = 0.0
    bad[1, 1, 4] = np.nan                                                  # the rotation is not scripted: not read
    e.set_rigid_script(bad)
    e.set_rigid_motion([])
    e.close()


def test_graph_replay_after_particles_are_deleted_and_appended_past_the_id_capacity():
    # a frame replayed from graphs, then the device edits: deleting the particles inside the floor and appending as many new
    # ones numbers them past the capacity of the by-id colour arrays, which are reallocated (as are the captured graphs that
    # held them); the next frame, replayed again, agrees with launches from the host
    runs = []
    for no_graph in (False, True):
        m = _paddle_scene(no_graph=no_graph, sunk=True)
        n0 = m._n_uploaded
        m._rigid_substeps(10)
        m.delete_particles_inside_level_set()
        k = n0 - m.num_particles()
        assert k > 100
        m.add_particles(type="jelly", positions=_layer(0.5)[:k], density=400.0, E=2e4)
        assert m._id_range() == n0 + k                            # ids past every id the colour arrays were sized for
        m._rigid_substeps(10)
        runs.append((m, k, m.engine.get_particle_cdf(n0 + k), m.get_particles()))
    (a, ka, ca, pa), (b, kb, cb, pb) = runs
    assert ka == kb and np.array_equal(pa["id"], pb["id"])
    assert np.abs(pa["x"] - pb["x"]).max() <= 1e-5 and np.abs(pa["v"] - pb["v"]).max() <= 1e-3 * np.abs(pb["v"]).max()
    assert (ca["states"] != cb["states"]).mean() <= 0.002 and (ca["states"] != 0).sum() > 20
    assert np.array_equal(ca["near"] != 0, cb["near"] != 0) or (ca["near"] != cb["near"]).mean() <= 0.002
    for j in range(2):
        assert np.abs(a.rigids[j].position - b.rigids[j].position).max() <= 1e-5


def test_levelset_collision_without_a_level_set_collides_with_nothing():
    # asked for but no level set (never set, or removed after contacts were found): the bodies move as without the collision
    runs = {}
    for name, floor, collide in (("off", None, False), ("no_levelset", None, True), ("removed", 0.25, True)):
        e, body, _ = _box_engine(dt=1e-3, particles=False, y=0.27, floor=floor, collide=collide)
        e.substep(1)                                              # "removed": the box starts inside the floor and collides
        start = rigid_mod.state_records([body])
        rs = e.get_rigid_state(2)
        start["position"][1], start["velocity"][1], start["angular_velocity"][1] = rs["position"][1], rs["velocity"][1], rs["angular_velocity"][1]
        start["rot"][1] = rs["rotation"][1].T.reshape(9)
        runs[name] = (e, start)
    ref = runs["removed"][1]                                      # every run continues from this state
    out = {}
    for name, (e, _) in runs.items():
        if name == "removed":
            e.set_sdf(None, 0.0)
        e.set_rigid_state(ref)
        e.substep(20)
        out[name] = e.get_rigid_state(2)
        e.close()
    for name in ("no_levelset", "removed"):
        for key in ("position", "velocity", "angular_velocity", "rotation"):
            assert np.array_equal(out[name][key], out["off"][key]), (name, key)
